// gemm.cu -- the dense-contraction workhorse: OUT[n, :] = act(scale * (A[n, :] @ W) + shift (+ res))
// where the A row of output row n is GATHERED on the fly:
//   rows mode : concat of up to 3 sources, each optionally gathered through an index
//               (nearest_interpolation / closest_pool / skip concat fused into the GEMM)
//   conv mode : the 9 taps of a 3x3 NHWC convolution (implicit GEMM, zero padding)
// and the result can be written row-major, NCHW, or pixel-shuffled (k == stride deconv).
//
// Replaces (reference, /root/reference/ml3d/torch/models):
//   SharedMLP (1x1 Conv2d/ConvTranspose2d + BN + LeakyReLU)      randlanet.py:471-518
//   fc0/bn0, decoder concat + SharedMLP, fc1                      randlanet.py:266-298
//   nearest_interpolation                                         randlanet.py:329-350
//   UnaryBlock / BatchNormBlock / closest_pool                    kpconv.py:1213-1295, 821-837
//   the [15*Cin, Cout] contraction of KPConv.forward              kpconv.py:1147-1159
//   SECOND / SECONDFPN / Anchor3DHead convolutions                point_pillars.py:619-841
//
// This file is the FP32 SIMT implementation (exact to ~1e-6 of the reference);
// register-tiled 8x4 per thread, BK = 16, register prefetch of the next k-tile.
#include "../../include/o3dml_b200.h"
#include "dense.cuh"

namespace o3dml {

constexpr int GEMM_THREADS = 256;
constexpr int GEMM_BK = 16;
constexpr int GEMM_TM = 8;
constexpr int GEMM_TN = 4;
constexpr int MAX_SRC = 3;

struct GemmParams {
    int64_t N;
    int K, Cout;
    int mode;  // 0 rows, 1 conv3x3
    int nsrc;
    o3dml_src_t src[MAX_SRC];
    int koff[MAX_SRC + 1];
    int vec_a;  // all sources float4-loadable
    // conv3x3 (src[0].data = NHWC input)
    int H, W, OH, OW, stride, C;
    const float* Wt;  // [K, Cout]
    DenseEpilogue ep;
};

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS)
gemm_gather_kernel(const __grid_constant__ GemmParams p) {
    constexpr int TX = BN / GEMM_TN;           // threads along N
    constexpr int TY = GEMM_THREADS / TX;      // threads along M
    constexpr int BM = TY * GEMM_TM;
    constexpr int A_F4 = BM * GEMM_BK / 4 / GEMM_THREADS;  // float4 per thread per k-tile
    constexpr int B_F4 = (BN * GEMM_BK / 4 + GEMM_THREADS - 1) / GEMM_THREADS;
    __shared__ __align__(16) float As[GEMM_BK][BM + 4];
    __shared__ __align__(16) float Bs[GEMM_BK][BN];
    __shared__ const float* rowptr[MAX_SRC][BM];  // rows mode: per-source row base
    __shared__ int rowinfo[BM][3];                // conv mode: image base pixel, iy0, ix0

    const DenseEpilogue& ep = p.ep;
    const int tid = threadIdx.x;
    const int tx = tid % TX, ty = tid / TX;
    const int64_t row0 = (int64_t)blockIdx.x * BM;
    const int col0 = blockIdx.y * BN;

    // ---- per-row gather bookkeeping, once per block
    if (p.mode == 0) {
        for (int i = tid; i < p.nsrc * BM; i += GEMM_THREADS) {
            int s = i / BM, m = i % BM;
            int64_t n = row0 + m;
            rowptr[s][m] = (n < p.N) ? src_row(p.src[s], n) : nullptr;
        }
    } else {
        for (int m = tid; m < BM; m += GEMM_THREADS) {
            int64_t n = row0 + m;
            if (n < p.N) {
                int64_t per = (int64_t)p.OH * p.OW;
                int b = (int)(n / per);
                int r = (int)(n % per);
                int oy = r / p.OW, ox = r % p.OW;
                rowinfo[m][0] = b * p.H * p.W;
                rowinfo[m][1] = oy * p.stride - 1;
                rowinfo[m][2] = ox * p.stride - 1;
            } else {
                rowinfo[m][0] = -1;
                rowinfo[m][1] = rowinfo[m][2] = 0;
            }
        }
    }
    __syncthreads();

    float acc[GEMM_TM][GEMM_TN];
#pragma unroll
    for (int i = 0; i < GEMM_TM; ++i)
#pragma unroll
        for (int j = 0; j < GEMM_TN; ++j) acc[i][j] = 0.f;

    float4 a_reg[A_F4];
    float4 b_reg[B_F4];
    const int ktiles = (p.K + GEMM_BK - 1) / GEMM_BK;

    auto load_tile = [&](int kt) {
        const int kbase = kt * GEMM_BK;
        // ---- A
#pragma unroll
        for (int i = 0; i < A_F4; ++i) {
            int f = tid + i * GEMM_THREADS;
            int m = f >> 2, kq = f & 3;
            int k = kbase + kq * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.mode == 1) {
                if (k < p.K && rowinfo[m][0] >= 0) {
                    int tap = k / p.C, c = k - tap * p.C;
                    int iy = rowinfo[m][1] + tap / 3, ix = rowinfo[m][2] + tap % 3;
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
                        v = *reinterpret_cast<const float4*>(
                            p.src[0].data + ((size_t)rowinfo[m][0] + (size_t)iy * p.W + ix) * p.C + c);
                }
            } else if (p.vec_a) {
                if (k < p.K) {
                    int s = 0;
                    while (s + 1 < p.nsrc && k >= p.koff[s + 1]) ++s;
                    const float* base = rowptr[s][m];
                    if (base) v = *reinterpret_cast<const float4*>(base + (k - p.koff[s]));
                }
            } else {
                float e[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    int kk = k + q;
                    e[q] = 0.f;
                    if (kk < p.K) {
                        int s = 0;
                        while (s + 1 < p.nsrc && kk >= p.koff[s + 1]) ++s;
                        const float* base = rowptr[s][m];
                        if (base) e[q] = base[kk - p.koff[s]];
                    }
                }
                v = make_float4(e[0], e[1], e[2], e[3]);
            }
            a_reg[i] = v;
        }
        // ---- B
#pragma unroll
        for (int i = 0; i < B_F4; ++i) {
            int f = tid + i * GEMM_THREADS;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (f < BN * GEMM_BK / 4) {
                int kk = f / (BN / 4), j = (f % (BN / 4)) * 4;
                int k = kbase + kk, col = col0 + j;
                if (k < p.K) {
                    const float* w = p.Wt + (size_t)k * p.Cout + col;
                    if ((p.Cout & 3) == 0 && col + 3 < p.Cout) {
                        v = *reinterpret_cast<const float4*>(w);
                    } else {
                        if (col + 0 < p.Cout) v.x = w[0];
                        if (col + 1 < p.Cout) v.y = w[1];
                        if (col + 2 < p.Cout) v.z = w[2];
                        if (col + 3 < p.Cout) v.w = w[3];
                    }
                }
            }
            b_reg[i] = v;
        }
    };
    auto store_tile = [&]() {
#pragma unroll
        for (int i = 0; i < A_F4; ++i) {
            int f = tid + i * GEMM_THREADS;
            int m = f >> 2, kq = f & 3;
            As[kq * 4 + 0][m] = a_reg[i].x;
            As[kq * 4 + 1][m] = a_reg[i].y;
            As[kq * 4 + 2][m] = a_reg[i].z;
            As[kq * 4 + 3][m] = a_reg[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_F4; ++i) {
            int f = tid + i * GEMM_THREADS;
            if (f < BN * GEMM_BK / 4) {
                int kk = f / (BN / 4), j = (f % (BN / 4)) * 4;
                *reinterpret_cast<float4*>(&Bs[kk][j]) = b_reg[i];
            }
        }
    };

    load_tile(0);
    for (int kt = 0; kt < ktiles; ++kt) {
        store_tile();
        __syncthreads();
        if (kt + 1 < ktiles) load_tile(kt + 1);
#pragma unroll
        for (int kk = 0; kk < GEMM_BK; ++kk) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * GEMM_TM]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * GEMM_TM + 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * GEMM_TN]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < GEMM_TM; ++i)
#pragma unroll
                for (int j = 0; j < GEMM_TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue
    const int cbase = col0 + tx * GEMM_TN;
    float sc[GEMM_TN], sh[GEMM_TN];
#pragma unroll
    for (int j = 0; j < GEMM_TN; ++j) {
        int c = cbase + j;
        sc[j] = (ep.scale && c < p.Cout) ? ep.scale[c] : 1.f;
        sh[j] = (ep.shift && c < p.Cout) ? ep.shift[c] : 0.f;
    }
#pragma unroll
    for (int i = 0; i < GEMM_TM; ++i) {
        const int64_t n = row0 + ty * GEMM_TM + i;
        if (n >= p.N) continue;
        float v[GEMM_TN];
#pragma unroll
        for (int j = 0; j < GEMM_TN; ++j) {
            int c = cbase + j;
            float x = fmaf(acc[i][j], sc[j], sh[j]);
            if (ep.residual && c < p.Cout) x += ep.residual[(size_t)n * ep.res_ld + c];
            v[j] = apply_act(x, ep.act, ep.slope);
        }
        if (ep.mode == 0 && cbase + 3 < p.Cout && (ep.out_ld & 3) == 0 &&
            ((reinterpret_cast<uintptr_t>(ep.out) & 15) == 0)) {
            *reinterpret_cast<float4*>(ep.out + out_offset(ep, n, cbase, p.Cout)) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < GEMM_TN; ++j)
                if (cbase + j < p.Cout) ep.out[out_offset(ep, n, cbase + j, p.Cout)] = v[j];
        }
    }
}

static int gemm_launch(GemmParams& p, cudaStream_t st) {
    if (p.N <= 0 || p.Cout <= 0) return O3DML_OK;
    p.vec_a = 1;
    for (int s = 0; s < p.nsrc; ++s)
        if ((p.src[s].channels & 3) || (p.src[s].ld & 3) || (reinterpret_cast<uintptr_t>(p.src[s].data) & 15)) p.vec_a = 0;
    // widest column tile that the output fills; narrow outputs get the tall tile
    if (p.Cout <= 32) {
        dim3 grid((unsigned)ceil_div<int64_t>(p.N, 256), (unsigned)ceil_div(p.Cout, 32));
        O3DML_CUDA(launch<gemm_gather_kernel<32>>(grid, GEMM_THREADS, 0, st, p));
    } else if (p.Cout <= 64 || p.N >= 4096) {
        dim3 grid((unsigned)ceil_div<int64_t>(p.N, 128), (unsigned)ceil_div(p.Cout, 64));
        O3DML_CUDA(launch<gemm_gather_kernel<64>>(grid, GEMM_THREADS, 0, st, p));
    } else {
        dim3 grid((unsigned)ceil_div<int64_t>(p.N, 64), (unsigned)ceil_div(p.Cout, 128));
        O3DML_CUDA(launch<gemm_gather_kernel<128>>(grid, GEMM_THREADS, 0, st, p));
    }
    return O3DML_OK;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_linear(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs,
                            const float* weight_t, const float* scale, const float* shift,
                            const float* residual, int residual_ld, int act, float slope,
                            float* out, int out_ld, int out_channels, int out_nchw_plane,
                            void* stream) {
    GemmParams p = {};
    p.N = num_rows;
    p.mode = 0;
    p.nsrc = num_srcs;
    p.Wt = weight_t;
    int rc = set_srcs("linear", srcs, num_srcs, p.src, p.koff);
    if (!rc) rc = set_epilogue("linear", p, weight_t, scale, shift, residual, residual_ld, act, slope, out, out_ld,
                               out_channels, out_nchw_plane);
    if (rc) return rc;
    p.K = p.koff[MAX_SRC];
    return gemm_launch(p, (cudaStream_t)stream);
}

extern "C" int o3dml_conv3x3_nhwc(const float* in, int batch, int H, int W, int C, int stride,
                                  const float* weight_t, const float* scale, const float* shift,
                                  int act, float slope, float* out, int out_channels, void* stream) {
    GemmParams p = {};
    p.Wt = weight_t;
    int rc = set_conv3x3("conv3x3", p, in, batch, H, W, C, stride, 16);
    if (!rc) rc = set_epilogue("conv3x3", p, weight_t, scale, shift, nullptr, 0, act, slope, out, out_channels,
                               out_channels, 0);
    if (rc) return rc;
    return gemm_launch(p, (cudaStream_t)stream);
}

extern "C" int o3dml_deconv_nhwc(const float* in, int batch, int H, int W, int C, int stride,
                                 const float* weight_t, const float* scale, const float* shift,
                                 int act, float slope, float* out, int out_ld, int out_channels,
                                 void* stream) {
    GemmParams p = {};
    p.Wt = weight_t;
    int rc = set_deconv("deconv", p, weight_t, in, batch, H, W, C, stride, scale, shift, act, slope, out, out_ld,
                        out_channels);
    if (rc) return rc;
    return gemm_launch(p, (cudaStream_t)stream);
}
