// rowmlp.cu -- narrow per-point dense layers (K <= 64 inputs, <= 64 outputs), one THREAD per row.
//
// These are the SharedMLPs of RandLA-Net's first level and classifier (randlanet.py:471-518 as
// used at :110-113, :653-664, :284-292): 360 k rows per step, 8..64 channels.  Their arithmetic
// intensity is 2*K*Cout / (4*(K + Cout)) <= 11 flop/B: HBM-bound layers.  The tiled kernels
// (gemm.cu, gemm_tc.cu) spend their time in per-CTA set-up and barrier phases at these widths,
// not in moving the few bytes per row these layers need.  Here a thread loads its
// input row (contiguous, consecutive lanes = consecutive rows), keeps it in registers, and
// multiplies by a weight matrix that travels in the KERNEL PARAMETER block: every FFMA takes its
// weight from the constant bank (LDCU.128 + FFMA with a uniform-register operand), so no shared
// memory, no barrier and no weight traffic at all.  Sources may be a concat of two tensors, the
// second optionally gathered through an index (decoder: nearest_interpolation).
#include "../../include/o3dml_b200.h"
#include "dense.cuh"
#include <string.h>

namespace o3dml {

template <int C0, int C1, int COUT>
struct alignas(16) RowMlpParams {
    static constexpr int K = C0 + C1;
    static constexpr int CP = (COUT + 3) & ~3;    // padded weight row: 16-byte constant loads
    o3dml_src_t src[2];
    int64_t N;
    float* out;
    int32_t out_ld, act;
    float slope;
    int32_t pad;
    float w[K * CP + 2 * CP];                     // [K][CP] weight, then scale[CP], shift[CP]
};

template <int C>
__device__ __forceinline__ void load_row(const float* p, float* x) {
    if (p == nullptr) {
#pragma unroll
        for (int i = 0; i < C; ++i) x[i] = 0.f;
    } else if (C % 4 == 0) {
#pragma unroll
        for (int i = 0; i < C / 4; ++i) {
            const float4 v = *reinterpret_cast<const float4*>(p + 4 * i);
            x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < C; ++i) x[i] = p[i];
    }
}

template <int C0, int C1, int COUT>
__global__ void __launch_bounds__(256)
rowmlp_kernel(const __grid_constant__ RowMlpParams<C0, C1, COUT> p) {
    using P = RowMlpParams<C0, C1, COUT>;
    constexpr int K = P::K, CP = P::CP;
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= p.N) return;
    float x[K];
    load_row<C0>(src_row(p.src[0], n), x);
    if (C1 > 0) load_row<C1>(src_row(p.src[1], n), x + C0);
    float acc[CP];
#pragma unroll
    for (int c = 0; c < CP; ++c) acc[c] = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int c = 0; c < CP; ++c) acc[c] = fmaf(x[k], p.w[k * CP + c], acc[c]);
#pragma unroll
    for (int c = 0; c < CP; ++c)
        acc[c] = apply_act(fmaf(acc[c], p.w[K * CP + c], p.w[K * CP + CP + c]), p.act, p.slope);
    float* o = p.out + (size_t)n * p.out_ld;
    if (COUT % 4 == 0) {
#pragma unroll
        for (int c = 0; c < COUT; c += 4)
            *reinterpret_cast<float4*>(o + c) = make_float4(acc[c], acc[c + 1], acc[c + 2], acc[c + 3]);
    } else {
#pragma unroll
        for (int c = 0; c < COUT; ++c) o[c] = acc[c];
    }
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int C0, int C1, int COUT>
static int rowmlp_launch(int64_t num_rows, const o3dml_src_t (&srcs)[2], const float* hw, const float* hs,
                         const float* ht, int act, float slope, float* out, int out_ld, cudaStream_t st) {
    using P = RowMlpParams<C0, C1, COUT>;
    static_assert(sizeof(P) <= 32000, "kernel parameter block too large");
    P p;
    memset(&p, 0, sizeof(p));
    for (int s = 0; s < (C1 > 0 ? 2 : 1); ++s) {
        const int c = s == 0 ? C0 : C1;
        O3DML_CHECK(srcs[s].channels == c, "linear_rows_small: source %d has %d channels, kernel expects %d", s,
                    srcs[s].channels, c);
        if (c % 4 == 0)
            O3DML_CHECK(aligned16(srcs[s].data) && srcs[s].ld % 4 == 0,
                        "linear_rows_small: source %d is not 16-byte aligned", s);
        p.src[s] = srcs[s];
    }
    if (COUT % 4 == 0)
        O3DML_CHECK(aligned16(out) && out_ld % 4 == 0, "linear_rows_small: output is not 16-byte aligned");
    p.N = num_rows;
    p.out = out;
    p.out_ld = out_ld;
    p.act = act;
    p.slope = slope;
    constexpr int K = P::K, CP = P::CP;
    for (int k = 0; k < K; ++k)
        for (int c = 0; c < COUT; ++c) p.w[k * CP + c] = hw[(size_t)k * COUT + c];
    for (int c = 0; c < COUT; ++c) {
        p.w[K * CP + c] = hs ? hs[c] : 1.f;
        p.w[K * CP + CP + c] = ht ? ht[c] : 0.f;
    }
    rowmlp_kernel<C0, C1, COUT><<<(unsigned)ceil_div<int64_t>(num_rows, 256), 256, 0, st>>>(p);
    O3DML_LAUNCH_CHECK();
    o3dml_count_launches(1);
    return O3DML_OK;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_linear_rows_small_supported(int c0, int c1, int out_channels) {
#define RM_CASE(A, B, C) if (c0 == A && c1 == B && out_channels == C) return 1;
#include "rowmlp_shapes.inc"
#undef RM_CASE
    return 0;
}

extern "C" int o3dml_linear_rows_small(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs,
                                       const float* h_weight_t, const float* h_scale,
                                       const float* h_shift, int act, float slope, float* out, int out_ld,
                                       int out_channels, void* stream) {
    O3DML_CHECK(num_rows >= 0 && srcs && (num_srcs == 1 || num_srcs == 2), "linear_rows_small: bad arguments");
    O3DML_CHECK(h_weight_t && out, "linear_rows_small: null weight / output");
    O3DML_CHECK(out_ld >= out_channels, "linear_rows_small: out_ld < out_channels");
    for (const void* hp : {(const void*)h_weight_t, (const void*)h_scale, (const void*)h_shift}) {
        if (!hp) continue;
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, hp) == cudaSuccess)
            O3DML_CHECK(attr.type != cudaMemoryTypeDevice, "linear_rows_small: weights must be in HOST memory");
        else
            cudaGetLastError();
    }
    o3dml_src_t src[2] = {};
    int koff[3];
    int rc = set_srcs("linear_rows_small", srcs, num_srcs, src, koff);
    if (rc) return rc;
    if (num_rows == 0) return O3DML_OK;
    const int c0 = src[0].channels, c1 = num_srcs == 2 ? src[1].channels : 0;
    cudaStream_t st = (cudaStream_t)stream;
#define RM_CASE(A, B, C)                                                                              \
    if (c0 == A && c1 == B && out_channels == C)                                                      \
        return rowmlp_launch<A, B, C>(num_rows, src, h_weight_t, h_scale, h_shift, act, slope, out, \
                                      out_ld, st);
#include "rowmlp_shapes.inc"
#undef RM_CASE
    O3DML_FAIL(O3DML_ERR_UNSUPPORTED, "linear_rows_small: shape (%d + %d) -> %d is not instantiated", c0, c1,
               out_channels);
}
