// rl_tail.cu -- the per-point tail of RandLA-Net as ONE kernel: the last decoder layer and the classifier
//   decoder[-1]  SharedMLP(transpose) on [skip | nearest_interpolation(x)]   (randlanet.py:284-292, 329-350)
//   fc1          SharedMLP 32->64, SharedMLP 64->32, Dropout (eval: identity), SharedMLP 32->classes   (randlanet.py:110-113, 294-298)
// chained through shared memory and the Hopper tensor cores.  As four row-per-thread launches these layers re-read their
// 8 KB weight blocks for every row and write every intermediate activation to HBM.
//
// Per 128-row tile (one warpgroup of 128 threads):
//   load the 32 + 32 input channels of the row (thread = row; skip row; coarse row through the interpolation index)
//   into the activation tile in shared memory, then for each layer:
//     the warpgroup reads the TF32 A fragments of rows 0-63 and 64-127 from the tile, splits them into hi / lo in
//     registers and issues K/8 x 3 register-A wgmma per half against the layer's resident weight image in shared
//     memory (3xTF32: Ah*Wh + Ah*Wl + Al*Wh, as gemm_tc.cu); folded BN / bias + LeakyReLU on the accumulators,
//     written back into the activation tile as the next layer's input
//   logits staged in shared memory, written as one contiguous, fully coalesced block (128 rows x classes floats).
// Activations never touch HBM between the four layers: 256 B in, 4 x classes B out per point.
// Weights: host-packed image (open3d_ml_b200._lib.pack_tail_image): per layer, per 32-wide k-chunk, hi then lo tiles of
// [N rows][32 floats] in the K-major SWIZZLE_128B layout, copied once per CTA with one cp.async.bulk.
#include "../../include/o3dml_b200.h"
#include "dense.cuh"
#include "tc.cuh"
#include <string.h>
#include <algorithm>

namespace o3dml {

constexpr int RT_THREADS = 128;
constexpr int RT_K1 = 64, RT_N1 = 32, RT_N2 = 64, RT_N3 = 32, RT_N4 = 32;   // 32+32 -> 32 -> 64 -> 32 -> classes (<= 32)
constexpr int RT_W1 = 0, RT_W2 = 16384, RT_W3 = 32768, RT_W4 = 49152, RT_WBYTES = 57344;
constexpr int RT_LD = RT_K1 + 4;     // activation tile row stride (floats): the fragment reads hit 32 banks
constexpr size_t RT_SMEM = RT_WBYTES + RT_THREADS * RT_LD * 4 + 64 + 1024;

struct RlTailParams {
    const float* skip;
    o3dml_src_t coarse;   // gathered through the interpolation index
    int skip_ld, classes;
    int64_t N;
    const float* wimg;
    float* out;
    float slope;
    float scale[4][64];
    float shift[4][64];
};

// D[128 x N] = act[128 x K] * W[K x N] as two 64-row wgmma halves (W image at wbase: per 32-wide k-chunk hi tiles
// first, then lo tiles); the activation tile is read once per 32-channel chunk, split into TF32 hi / lo in registers
template <int K, int N>
__device__ __forceinline__ void rt_layer(const float* act, uint32_t wbase, float (*d)[N / 2], int tid) {
    constexpr int CHUNKS = K / 32;
    constexpr uint32_t TILE = N * 128;                       // bytes of one [N x 32 floats] tile
    const int lane = tid & 31, t = lane & 3;
    const int rw = (tid >> 5) * 16 + (lane >> 2);            // fragment rows rw, rw + 8 of each half
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = h * 64 + rw + (e & 1) * 8, k = c * 32 + ks * 8 + t + (e >> 1) * 4;
                    tc::split_tf32(__float_as_uint(act[r * RT_LD + k]), ah[ks][e], al[ks][e]);
                }
            tc::wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const uint64_t bh = tc::smem_desc_sw128(wbase + c * TILE + ks * 32);
                const uint64_t bl = tc::smem_desc_sw128(wbase + (CHUNKS + c) * TILE + ks * 32);
                tc::wgmma_tf32_rs<N>(d[h], ah[ks], bh, (c | ks) != 0);
                tc::wgmma_tf32_rs<N>(d[h], ah[ks], bl, 1u);
                tc::wgmma_tf32_rs<N>(d[h], al[ks], bh, 1u);
            }
            tc::wgmma_commit();
            tc::wgmma_wait_all();
        }
    }
}

// accumulators of the layer -> folded BN / bias (+ LeakyReLU) -> activation tile (row stride ld)
template <int N, bool ACT>
__device__ __forceinline__ void rt_store_d(const float (*d)[N / 2], const RlTailParams& p, int layer, float* act, int ld,
                                           int ncols, int tid) {
    const int lane = tid & 31, t = lane & 3;
    const int rw = (tid >> 5) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const int r = h * 64 + rw + ((i >> 1) & 1) * 8, c = (i >> 2) * 8 + 2 * t + (i & 1);
            float y = fmaf(d[h][i], p.scale[layer][c], p.shift[layer][c]);
            if (ACT) y = y >= 0.f ? y : y * p.slope;
            if (c < ncols) act[r * ld + c] = y;
        }
}

__global__ void __launch_bounds__(RT_THREADS, 2) rl_tail_kernel(const __grid_constant__ RlTailParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = tc::smem_u32(smem_raw);
    uint8_t* wsm = smem_raw + ((1024u - (raw & 1023u)) & 1023u);
    float* act = reinterpret_cast<float*>(wsm + RT_WBYTES);                 // [128][RT_LD] activations / logits of the tile
    uint64_t* mbar = reinterpret_cast<uint64_t*>(act + RT_THREADS * RT_LD);  // weights landed
    const int tid = threadIdx.x;
    if (tid == 0) {
        tc::mbar_init(&mbar[0], 1);
        tc::fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) {
        tc::mbar_arrive_expect_tx(&mbar[0], RT_WBYTES);
        tc::bulk_copy_g2s(wsm, p.wimg, RT_WBYTES, &mbar[0]);
    }
    const uint32_t wbase = tc::smem_u32(wsm);
    tc::mbar_wait(&mbar[0], 0);
    const int64_t tiles = ceil_div<int64_t>(p.N, RT_THREADS);
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t n = tile * RT_THREADS + tid;
        // ---- layer-1 operand: [skip row | interpolated coarse row]
        const float* s0 = nullptr;
        const float* s1 = nullptr;
        if (n < p.N) {
            s0 = p.skip + (size_t)n * p.skip_ld;
            s1 = src_row(p.coarse, n);
        }
        float4* arow = reinterpret_cast<float4*>(act + tid * RT_LD);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            arow[i] = s0 ? *reinterpret_cast<const float4*>(s0 + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
            arow[8 + i] = s1 ? *reinterpret_cast<const float4*>(s1 + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
        {   // ---- decoder[-1]: 64 -> 32
            float d[2][RT_N1 / 2];
            rt_layer<RT_K1, RT_N1>(act, wbase + RT_W1, d, tid);
            __syncthreads();
            rt_store_d<RT_N1, true>(d, p, 0, act, RT_LD, RT_N1, tid);
            __syncthreads();
        }
        {   // ---- fc1.0: 32 -> 64
            float d[2][RT_N2 / 2];
            rt_layer<RT_N1, RT_N2>(act, wbase + RT_W2, d, tid);
            __syncthreads();
            rt_store_d<RT_N2, true>(d, p, 1, act, RT_LD, RT_N2, tid);
            __syncthreads();
        }
        {   // ---- fc1.1: 64 -> 32
            float d[2][RT_N3 / 2];
            rt_layer<RT_N2, RT_N3>(act, wbase + RT_W3, d, tid);
            __syncthreads();
            rt_store_d<RT_N3, true>(d, p, 2, act, RT_LD, RT_N3, tid);
            __syncthreads();
        }
        {   // ---- fc1.3: 32 -> classes (no BN, no activation); logits as a dense [rows x classes] block
            float d[2][RT_N4 / 2];
            rt_layer<RT_N3, RT_N4>(act, wbase + RT_W4, d, tid);
            __syncthreads();
            rt_store_d<RT_N4, false>(d, p, 3, act, p.classes, p.classes, tid);
            __syncthreads();
        }
        const int64_t rows = min((int64_t)RT_THREADS, p.N - tile * RT_THREADS);
        float* o = p.out + (size_t)tile * RT_THREADS * p.classes;
        for (int i = tid; i < (int)(rows * p.classes); i += RT_THREADS) o[i] = act[i];
        __syncthreads();        // the activation tile is free for the next tile
    }
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_randla_tail_supported(int skip_channels, int coarse_channels, int c1, int c2, int c3, int classes) {
    return skip_channels == 32 && coarse_channels == 32 && c1 == RT_N1 && c2 == RT_N2 && c3 == RT_N3 && classes >= 1 &&
           classes <= RT_N4;
}

extern "C" int o3dml_randla_tail(const float* skip, int skip_ld, const float* coarse, int coarse_ld, int64_t coarse_rows,
                                 const void* interp_index, int index_is64, int64_t out_rows_per_batch,
                                 int64_t src_rows_per_batch, int64_t num_rows, const void* weight_image,
                                 const float* h_scale, const float* h_shift, float slope, int classes, float* out,
                                 void* stream) {
    O3DML_CHECK(skip && coarse && interp_index && weight_image && h_scale && h_shift && out, "randla_tail: null argument");
    O3DML_CHECK(classes >= 1 && classes <= RT_N4, "randla_tail: 1..32 classes");
    O3DML_CHECK((skip_ld & 3) == 0 && (coarse_ld & 3) == 0 && (reinterpret_cast<uintptr_t>(skip) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(coarse) & 15) == 0 && (reinterpret_cast<uintptr_t>(weight_image) & 15) == 0,
                "randla_tail: 16-byte aligned rows and weight image");
    if (num_rows <= 0) return O3DML_OK;
    RlTailParams p;
    p.skip = skip; p.skip_ld = skip_ld; p.classes = classes; p.N = num_rows;
    p.coarse = {coarse, interp_index, coarse_rows, out_rows_per_batch, src_rows_per_batch, RT_K1 / 2, coarse_ld,
                index_is64, 1};
    p.wimg = (const float*)weight_image; p.out = out; p.slope = slope;
    memcpy(p.scale, h_scale, sizeof(p.scale));
    memcpy(p.shift, h_shift, sizeof(p.shift));
    const int64_t tiles = ceil_div<int64_t>(num_rows, RT_THREADS);
    const unsigned grid = (unsigned)std::min<int64_t>(tiles, (int64_t)device_sm_count() * 2);
    O3DML_CUDA(launch<rl_tail_kernel>(grid, RT_THREADS, RT_SMEM, (cudaStream_t)stream, p));
    return O3DML_OK;
}
