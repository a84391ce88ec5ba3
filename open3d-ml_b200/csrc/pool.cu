// pool.cu -- index-driven pooling kernels (pure gather traffic, HBM/L2-bound):
//   gather_max      : out[n,:] = max_j src[idx[n,j],:]   (RandLA random_sample, KPConv max_pool;
//                     k = 1 gives nearest_interpolation / closest_pool)
//   kpconv_gather   : A[n, k*Cin + c] = sum_h infl(n,k,h) * x[idx[n,h], c]
//                     the neighbour-gather + kernel-point correlation half of KPConv.forward;
//                     the [15*Cin, Cout] contraction that follows runs in gemm.cu.
//
// Replaces (reference /root/reference/ml3d/torch/models):
//   RandLANet.random_sample          randlanet.py:300-327
//   max_pool / closest_pool          kpconv.py:821-858
//   KPConv.forward (rigid, linear influence, sum aggregation)   kpconv.py:1044-1147
#include "../../include/o3dml_b200.h"
#include "common.cuh"
#include <float.h>

namespace o3dml {

__global__ void __launch_bounds__(256)
gather_max_kernel(const float* __restrict__ src, int64_t src_rows, int C, int ld,
                  const void* __restrict__ idx, int idx_is64, int64_t n, int k,
                  int64_t out_rows_per_batch, int64_t src_rows_per_batch, int shadow_zero,
                  float* __restrict__ out, int out_ld) {
    const int c4n = C >> 2;
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n * c4n) return;
    const int64_t row = t / c4n;
    const int c = (int)(t % c4n) * 4;
    const int64_t boff = out_rows_per_batch > 0 ? (row / out_rows_per_batch) * src_rows_per_batch : 0;
    const int64_t lim = out_rows_per_batch > 0 ? src_rows_per_batch : src_rows;
    float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);   // a max over -inf rows is -inf
    bool any = false;
    for (int j = 0; j < k; ++j) {
        const int64_t r = load_index(idx, row * k + j, idx_is64);
        float4 v;
        if (r < 0 || r >= lim) {
            if (!shadow_zero) continue;
            v = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            v = *reinterpret_cast<const float4*>(src + (size_t)(boff + r) * ld + c);
        }
        best.x = fmaxf(best.x, v.x); best.y = fmaxf(best.y, v.y);
        best.z = fmaxf(best.z, v.z); best.w = fmaxf(best.w, v.w);
        any = true;
    }
    if (!any) best = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(out + (size_t)row * out_ld + c) = best;
}

constexpr int KP_MAXK = 16;   // kernel points handled (reference configs use 15)

// One warp per query point.  Lane h (and h+32) computes the 15 influence weights of
// neighbour h; the warp then walks the neighbours, every lane accumulating its channels
// (NE channels per lane and pass: 1 for Cin <= 32, 2 for <= 64, 4 otherwise).
template <int NE>
__global__ void __launch_bounds__(256)
kpconv_gather_kernel(const float* __restrict__ q_pts, const float* __restrict__ s_pts,
                     int64_t n_support, const void* __restrict__ nidx, int idx_is64, int H,
                     const float* __restrict__ x, int Cin, const float* __restrict__ kpts, int K,
                     float extent, int64_t nq, float* __restrict__ out) {
    __shared__ float kp[KP_MAXK * 3];
    if (threadIdx.x < K * 3) kp[threadIdx.x] = kpts[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t q = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (q >= nq) return;
    const float qx = q_pts[3 * q], qy = q_pts[3 * q + 1], qz = q_pts[3 * q + 2];
    const float inv_ext = extent;  // divide, as the reference does
    const int KK = K * Cin;
    constexpr int KP_CCH = 32 * NE;
    for (int h0 = 0; h0 < H || h0 == 0; h0 += 32) {
        // ---- influence weights of neighbour h0+lane
        float w[KP_MAXK];
        int64_t nb = -1;
        if (h0 + lane < H) {
            nb = load_index(nidx, q * H + h0 + lane, idx_is64);
            if (nb < 0 || nb >= n_support) nb = -1;  // shadow neighbour: zero influence, zero feature
        }
#pragma unroll
        for (int k = 0; k < KP_MAXK; ++k) w[k] = 0.f;
        if (nb >= 0) {
            const float nx = s_pts[3 * nb] - qx, ny = s_pts[3 * nb + 1] - qy, nz = s_pts[3 * nb + 2] - qz;
#pragma unroll
            for (int k = 0; k < KP_MAXK; ++k) {
                if (k < K) {
                    const float dx = nx - kp[3 * k], dy = ny - kp[3 * k + 1], dz = nz - kp[3 * k + 2];
                    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                    w[k] = fmaxf(1.f - __fdiv_rn(sqrtf(d2), inv_ext), 0.f);
                }
            }
        }
        const int hcount = min(32, H - h0);
        // ---- accumulate channel chunks
        for (int c0 = 0; c0 < Cin; c0 += KP_CCH) {
            float acc[KP_MAXK][KP_CCH / 32];
#pragma unroll
            for (int k = 0; k < KP_MAXK; ++k)
#pragma unroll
                for (int e = 0; e < KP_CCH / 32; ++e) acc[k][e] = 0.f;
            for (int h = 0; h < hcount; ++h) {
                const int64_t nbh = __shfl_sync(0xffffffffu, nb, h);
                if (nbh < 0) continue;  // warp-uniform
                float xv[KP_CCH / 32];
#pragma unroll
                for (int e = 0; e < KP_CCH / 32; ++e) {
                    const int c = c0 + e * 32 + lane;
                    xv[e] = (c < Cin) ? x[(size_t)nbh * Cin + c] : 0.f;
                }
#pragma unroll
                for (int k = 0; k < KP_MAXK; ++k) {
                    const float wk = __shfl_sync(0xffffffffu, w[k], h);
#pragma unroll
                    for (int e = 0; e < KP_CCH / 32; ++e) acc[k][e] = fmaf(wk, xv[e], acc[k][e]);
                }
            }
            float* o = out + (size_t)q * KK;
#pragma unroll
            for (int k = 0; k < KP_MAXK; ++k) {
                if (k < K) {
#pragma unroll
                    for (int e = 0; e < KP_CCH / 32; ++e) {
                        const int c = c0 + e * 32 + lane;
                        if (c < Cin) {
                            if (h0 == 0) o[k * Cin + c] = acc[k][e];
                            else o[k * Cin + c] += acc[k][e];
                        }
                    }
                }
            }
        }
    }
}

// Group-per-query variant for Cin % 4 == 0 (every layer but the first): LPQ = 8 / 16 / 32 lanes
// own one query (4 / 2 / 1 queries per warp), 4 channels per lane.  The first version above
// broadcast every influence weight with a shuffle (17 SHFL per neighbour for 15 FMAs at Cin = 32:
// bound by the 32 lanes/clk shuffle datapath, 880 us for the 262 k-query layers of an S3DIS
// batch).  Here lane (q, h) computes the 15 influences of one (query, neighbour) pair of the
// current chunk of LPQ neighbours and parks them in shared memory; the accumulate loop then
// fetches 16 weights with 4 LDS.128 per neighbour and feeds 60 FMAs per lane from them, and the
// neighbour's feature row arrives as one float4 per lane (LPQ x 16 B contiguous).
//
// DEFORM (deformable KPConv, kpconv.py:1011-1106, modulated = False): every query has its own kernel
// points kp_k + extent * offsets[q, 3k .. 3k+2] (product and sum rounded separately, as the reference),
// parked per query in shared memory.  A neighbour is kept when d2 < extent^2 for at least one of
// them; the group compacts its kept neighbours in ascending row position (ballot + popc) into the
// w_s / nb_s slots, so a dropped neighbour costs neither a feature load nor an FMA.
template <int LPQ, int NE, bool DEFORM = false>   // NE channels per lane: 4 (float4 rows) or 1 (unaligned Cin <= 8)
__global__ void __launch_bounds__(256)
kpconv_gather_grouped_kernel(const float* __restrict__ q_pts, const float* __restrict__ s_pts,
                             int64_t n_support, const void* __restrict__ nidx, int idx_is64, int H,
                             const float* __restrict__ x, int Cin, const float* __restrict__ kpts, int K,
                             float extent, int64_t nq, float* __restrict__ out,
                             const float* __restrict__ offsets, int offset_ld) {
    constexpr int QPW = 32 / LPQ;                       // queries per warp
    __shared__ float4 kp4[(DEFORM ? 8 * QPW : 1) * KP_MAXK];   // DEFORM: [warp][query][kernel point]
    // [warp][4 kernel points][slot]: slot = row ^ (row / LPQ) spreads the QPW rows that are read
    // together (same neighbour position of the QPW queries) over different banks
    __shared__ float4 w_s[8][KP_MAXK / 4][32];
    __shared__ int nb_s[8][32];
    if constexpr (!DEFORM) {
        if (threadIdx.x < KP_MAXK)
            kp4[threadIdx.x] = threadIdx.x < K ? make_float4(kpts[3 * threadIdx.x], kpts[3 * threadIdx.x + 1],
                                                             kpts[3 * threadIdx.x + 2], 0.f)
                                               : make_float4(1e18f, 1e18f, 1e18f, 0.f);   // unused slot: weight 0
        __syncthreads();
    }
    const float inv_ext = 1.f / extent;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int qg = lane / LPQ, lq = lane % LPQ;          // query of this lane within the warp, lane within group
    const int64_t wq0 = ((int64_t)blockIdx.x * 8 + wib) * QPW;
    if (wq0 >= nq) return;                               // warp-uniform
    const int64_t q = wq0 + qg;
    const bool qok = q < nq;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (qok) { qx = q_pts[3 * q]; qy = q_pts[3 * q + 1]; qz = q_pts[3 * q + 2]; }
    float4* const kpw = kp4 + (DEFORM ? (wib * QPW + qg) * KP_MAXK : 0);   // this lane's kernel points
    float ext2 = 0.f;
    if constexpr (DEFORM) {
        ext2 = extent * extent;
        for (int k = lq; k < KP_MAXK; k += LPQ) {
            float4 d = make_float4(1e18f, 1e18f, 1e18f, 0.f);                  // unused slot: never in range
            if (qok && k < K) {
                const float* o = offsets + (size_t)q * offset_ld + 3 * k;
                d = make_float4(__fadd_rn(__fmul_rn(o[0], extent), kpts[3 * k]),
                                __fadd_rn(__fmul_rn(o[1], extent), kpts[3 * k + 1]),
                                __fadd_rn(__fmul_rn(o[2], extent), kpts[3 * k + 2]), 0.f);
            }
            kpw[k] = d;
        }
        __syncwarp();
    }
    const int KK = K * Cin;
    for (int c0 = 0; c0 < Cin; c0 += LPQ * NE) {
        const int c = c0 + NE * lq;
        float acc[KP_MAXK][NE];
#pragma unroll
        for (int k = 0; k < KP_MAXK; ++k)
#pragma unroll
            for (int e = 0; e < NE; ++e) acc[k][e] = 0.f;
        for (int h0 = 0; h0 < H; h0 += LPQ) {
            // ---- influences of (query qg, neighbour h0 + lq)
            int nb = -1;
            if (qok && h0 + lq < H) {
                const int64_t r = load_index(nidx, q * H + h0 + lq, idx_is64);
                if (r >= 0 && r < n_support) nb = (int)r;   // else shadow: zero influence, zero feature
            }
            // trailing all-shadow positions (the padded tail of the neighbour rows) are skipped for the
            // whole warp; hc = one past the last position that is valid for any of the QPW queries
            int hc = 0;
            if constexpr (!DEFORM) {
                const unsigned valid = __ballot_sync(0xffffffffu, nb >= 0);
                if (valid == 0u) continue;
#pragma unroll
                for (int g = 0; g < QPW; ++g) {
                    const unsigned mg = (LPQ == 32) ? valid : ((valid >> (g * LPQ)) & ((1u << (LPQ & 31)) - 1u));
                    hc = max(hc, 32 - __clz(mg));
                }
            }
            float w[KP_MAXK];
#pragma unroll
            for (int k = 0; k < KP_MAXK; ++k) w[k] = 0.f;
            bool keep = false;
            if (nb >= 0) {
                const float nx = s_pts[3 * (size_t)nb] - qx, ny = s_pts[3 * (size_t)nb + 1] - qy,
                            nz = s_pts[3 * (size_t)nb + 2] - qz;
#pragma unroll
                for (int k = 0; k < KP_MAXK; ++k) {      // linear influence max(0, 1 - |y - kp_k| / extent)
                    const float4 kk = DEFORM ? kpw[k] : kp4[k];
                    const float dx = nx - kk.x, dy = ny - kk.y, dz = nz - kk.z;
                    const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
                    if constexpr (DEFORM) keep |= d2 < ext2;
                    float dist;                          // 2-ulp sqrt: far inside the 1e-4 feature tolerance
                    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(dist) : "f"(d2));
                    w[k] = fmaxf(fmaf(-dist, inv_ext, 1.f), 0.f);
                }
            }
            // DEFORM: slot row of this lane's neighbour after compaction, and the group's kept count
            int row = lane, kept = 0;
            if constexpr (DEFORM) {
                const unsigned valid = __ballot_sync(0xffffffffu, keep);
                if (valid == 0u) continue;
                const unsigned mg = (LPQ == 32) ? valid : ((valid >> (qg * LPQ)) & ((1u << (LPQ & 31)) - 1u));
                kept = __popc(mg);
                row = qg * LPQ + __popc(mg & ((1u << lq) - 1u));
            }
            __syncwarp();                                   // previous chunk fully consumed
            if (!DEFORM || keep) {
#pragma unroll
                for (int k4 = 0; k4 < KP_MAXK / 4; ++k4)
                    w_s[wib][k4][row ^ qg] = make_float4(w[4 * k4], w[4 * k4 + 1], w[4 * k4 + 2], w[4 * k4 + 3]);
                nb_s[wib][row] = nb;
            }
            __syncwarp();
            // ---- accumulate the chunk: 4 channels per lane (DEFORM: the group's kept neighbours only)
            for (int hh = 0; hh < (DEFORM ? kept : hc); ++hh) {
                const int nbh = nb_s[wib][qg * LPQ + hh];
                float xv[NE];
#pragma unroll
                for (int e = 0; e < NE; ++e) xv[e] = 0.f;
                if (nbh >= 0 && c < Cin) {
                    if (NE == 4) {
                        const float4 t = *reinterpret_cast<const float4*>(x + (size_t)nbh * Cin + c);
                        xv[0] = t.x; xv[NE > 1 ? 1 : 0] = t.y; xv[NE > 2 ? 2 : 0] = t.z; xv[NE > 3 ? 3 : 0] = t.w;
                    } else {
                        xv[0] = x[(size_t)nbh * Cin + c];
                    }
                }
                const int slot = (qg * LPQ + hh) ^ qg;
#pragma unroll
                for (int k4 = 0; k4 < KP_MAXK / 4; ++k4) {
                    const float4 wv = w_s[wib][k4][slot];
                    const float wk[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int e = 0; e < NE; ++e) acc[4 * k4 + j][e] = fmaf(wk[j], xv[e], acc[4 * k4 + j][e]);
                }
            }
        }
        if (qok && c < Cin) {
            float* o = out + (size_t)q * KK + c;
#pragma unroll
            for (int k = 0; k < KP_MAXK; ++k) {
                if (k < K) {
                    if (NE == 4)
                        *reinterpret_cast<float4*>(o + (size_t)k * Cin) =
                            make_float4(acc[k][0], acc[k][NE > 1 ? 1 : 0], acc[k][NE > 2 ? 2 : 0], acc[k][NE > 3 ? 3 : 0]);
                    else
                        o[(size_t)k * Cin] = acc[k][0];
                }
            }
        }
    }
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_gather_max(const float* src, int64_t src_rows, int channels, int src_ld,
                                const void* index, int index_is64, int64_t num_rows, int k,
                                int64_t out_rows_per_batch, int64_t src_rows_per_batch,
                                int shadow_zero, float* out, int out_ld, void* stream) {
    O3DML_CHECK((channels & 3) == 0 && (src_ld & 3) == 0 && (out_ld & 3) == 0,
                "gather_max: channels and strides must be multiples of 4");
    O3DML_CHECK(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                "gather_max: buffers must be 16-byte aligned");
    O3DML_CHECK(k >= 1, "gather_max: k >= 1");
    if (num_rows <= 0) return O3DML_OK;
    int64_t total = num_rows * (channels / 4);
    O3DML_CUDA(launch<gather_max_kernel>((unsigned)ceil_div<int64_t>(total, 256), 256, 0, (cudaStream_t)stream, src,
                                         src_rows, channels, src_ld, index, index_is64, num_rows, k,
                                         out_rows_per_batch, src_rows_per_batch, shadow_zero, out, out_ld));
    return O3DML_OK;
}

extern "C" int o3dml_kpconv_gather(const float* query_points, int64_t num_queries,
                                   const float* support_points, int64_t num_support,
                                   const void* neighbor_index, int index_is64, int max_neighbors,
                                   const float* features, int in_channels,
                                   const float* kernel_points, int num_kernel_points,
                                   float kp_extent, float* weighted_features, void* stream) {
    O3DML_CHECK(num_kernel_points >= 1 && num_kernel_points <= KP_MAXK,
                "kpconv: at most %d kernel points", KP_MAXK);
    O3DML_CHECK(max_neighbors >= 0 && in_channels >= 1 && kp_extent > 0.f, "kpconv: bad sizes");
    if (num_queries <= 0) return O3DML_OK;
    const unsigned nb = (unsigned)ceil_div<int64_t>(num_queries, 8);
    cudaStream_t st = (cudaStream_t)stream;
    const bool aligned = (in_channels & 3) == 0 && num_support < ((int64_t)1 << 31) &&
                         ((reinterpret_cast<uintptr_t>(features) | reinterpret_cast<uintptr_t>(weighted_features)) & 15) == 0;
    const bool narrow = in_channels <= 8 && num_support < ((int64_t)1 << 31);
    if (aligned || narrow) {
#define KPG_LAUNCH(LPQ, NE)                                                                                        \
    O3DML_CUDA(launch<kpconv_gather_grouped_kernel<LPQ, NE>>(                                                      \
        (unsigned)ceil_div<int64_t>(num_queries, 8 * (32 / LPQ)), 256, 0, st, query_points, support_points,      \
        num_support, neighbor_index, index_is64, max_neighbors, features, in_channels, kernel_points,          \
        num_kernel_points, kp_extent, num_queries, weighted_features, nullptr, 0))
        if (!aligned) KPG_LAUNCH(8, 1);
        else if (in_channels <= 32) KPG_LAUNCH(8, 4);
        else if (in_channels <= 64) KPG_LAUNCH(16, 4);
        else KPG_LAUNCH(32, 4);
#undef KPG_LAUNCH
        return O3DML_OK;
    }
#define KP_LAUNCH(NE)                                                                                         \
    O3DML_CUDA(launch<kpconv_gather_kernel<NE>>(nb, 256, 0, st, query_points, support_points, num_support,    \
                                                neighbor_index, index_is64, max_neighbors, features,         \
                                                in_channels, kernel_points, num_kernel_points, kp_extent,    \
                                                num_queries, weighted_features))
    if (in_channels <= 32) KP_LAUNCH(1);
    else if (in_channels <= 64) KP_LAUNCH(2);
    else KP_LAUNCH(4);
#undef KP_LAUNCH
    return O3DML_OK;
}

extern "C" int o3dml_kpconv_gather_deformable(const float* query_points, int64_t num_queries,
                                              const float* support_points, int64_t num_support,
                                              const void* neighbor_index, int index_is64, int max_neighbors,
                                              const float* features, int in_channels,
                                              const float* kernel_points, int num_kernel_points,
                                              float kp_extent, const float* offsets, int offset_ld,
                                              float* weighted_features, void* stream) {
    O3DML_CHECK(num_kernel_points >= 1 && num_kernel_points <= KP_MAXK,
                "kpconv_deformable: at most %d kernel points", KP_MAXK);
    O3DML_CHECK(max_neighbors >= 0 && in_channels >= 1 && kp_extent > 0.f, "kpconv_deformable: bad sizes");
    O3DML_CHECK(offsets != nullptr && offset_ld >= 3 * num_kernel_points,
                "kpconv_deformable: offsets [num_queries, >= 3K] required");
    const bool aligned = (in_channels & 3) == 0 &&
                         ((reinterpret_cast<uintptr_t>(features) | reinterpret_cast<uintptr_t>(weighted_features)) & 15) == 0;
    O3DML_CHECK(num_support < ((int64_t)1 << 31) && (aligned || in_channels <= 8),
                "kpconv_deformable: Cin % 4 == 0 with 16-byte aligned rows, or Cin <= 8; fewer than 2^31 supports");
    if (num_queries <= 0) return O3DML_OK;
    cudaStream_t st = (cudaStream_t)stream;
#define KPD_LAUNCH(LPQ, NE)                                                                                        \
    O3DML_CUDA(launch<kpconv_gather_grouped_kernel<LPQ, NE, true>>(                                                \
        (unsigned)ceil_div<int64_t>(num_queries, 8 * (32 / LPQ)), 256, 0, st, query_points, support_points,      \
        num_support, neighbor_index, index_is64, max_neighbors, features, in_channels, kernel_points,          \
        num_kernel_points, kp_extent, num_queries, weighted_features, offsets, offset_ld))
    if (!aligned) KPD_LAUNCH(8, 1);
    else if (in_channels <= 32) KPD_LAUNCH(8, 4);
    else if (in_channels <= 64) KPD_LAUNCH(16, 4);
    else KPD_LAUNCH(32, 4);
#undef KPD_LAUNCH
    return O3DML_OK;
}
