// dense.cuh -- how the dense-layer kernels (gemm.cu, gemm_tc.cu, rowmlp.cu, rl_tail.cu) read a gathered operand and
// describe their output, and the host-side checks that go with both.
#pragma once
#include "../../include/o3dml_b200.h"
#include "common.cuh"

namespace o3dml {

// Address of row n of a source: row n itself, or the row its index names (global, or relative to batch item
// n / out_rows_per_batch).  nullptr for a row that reads as zeros: a negative id, a batch-relative id past
// src_rows_per_batch, or a resolved row outside [0, rows) (the shadow neighbours of KPConv).
__device__ __forceinline__ const float* src_row(const o3dml_src_t& S, int64_t n) {
    int64_t r = n;
    if (S.index) {
        r = load_index(S.index, n * S.index_ld, S.index_is64);
        if (r < 0) return nullptr;
        if (S.out_rows_per_batch > 0) {
            if (r >= S.src_rows_per_batch) return nullptr;
            r += (n / S.out_rows_per_batch) * S.src_rows_per_batch;
        }
        if (r >= S.rows) return nullptr;
    }
    return S.data + (size_t)r * S.ld;
}

// Checks 1..MAX sources (data, channels > 0, ld >= channels) and copies them into kernel parameters with index_ld <= 0
// read as 1.  koff[s] is the first k of source s; koff[num..MAX] = K, the summed channel count.
template <int MAX>
inline int set_srcs(const char* fn, const o3dml_src_t* srcs, int num, o3dml_src_t (&dst)[MAX], int (&koff)[MAX + 1]) {
    O3DML_CHECK(srcs && num >= 1 && num <= MAX, "%s: 1..%d sources", fn, MAX);
    int k = 0;
    for (int s = 0; s < num; ++s) {
        const o3dml_src_t& S = srcs[s];
        O3DML_CHECK(S.data && S.channels > 0 && S.ld >= S.channels, "%s: bad source %d", fn, s);
        dst[s] = S;
        dst[s].index_ld = S.index ? (S.index_ld > 0 ? S.index_ld : 1) : 0;
        koff[s] = k;
        k += S.channels;
    }
    for (int s = num; s <= MAX; ++s) koff[s] = k;
    return O3DML_OK;
}

// What the GEMM kernels do with an accumulated row: out = act(scale * acc + shift + residual), written row-major,
// as NCHW planes, or pixel-shuffled (the deconvolution with kernel == stride).
struct DenseEpilogue {
    const float* scale;
    const float* shift;
    const float* residual;
    int res_ld;
    int act;
    float slope;
    float* out;
    int out_ld;
    int mode;       // 0 rows, 1 NCHW, 2 deconv pixel shuffle
    int64_t plane;  // NCHW: rows per image
    int ds, dIH, dIW, dC;   // pixel shuffle: stride, input height and width, channels per sub-pixel
};

// Fills p.ep and p.Cout for a row-major (out_nchw_plane == 0) or NCHW output and checks them together with the weight
// operand the caller passes to its kernel.
template <class P>
inline int set_epilogue(const char* fn, P& p, const void* weight, const float* scale, const float* shift,
                        const float* residual, int residual_ld, int act, float slope, float* out, int out_ld,
                        int out_channels, int out_nchw_plane) {
    O3DML_CHECK(act >= 0 && act <= 2, "%s: unknown activation %d", fn, act);
    O3DML_CHECK(weight && out, "%s: null weight/out", fn);
    O3DML_CHECK((reinterpret_cast<uintptr_t>(weight) & 15) == 0, "%s: weight must be 16-byte aligned", fn);
    p.Cout = out_channels;
    DenseEpilogue& e = p.ep;
    e = {};
    e.scale = scale; e.shift = shift; e.residual = residual; e.res_ld = residual_ld;
    e.act = act; e.slope = slope; e.out = out; e.out_ld = out_ld;
    if (out_nchw_plane > 0) {
        e.mode = 1;
        e.plane = out_nchw_plane;
    }
    return O3DML_OK;
}

// A 3x3 convolution, padding 1, stride 1 or 2, over an NHWC input as an implicit GEMM: one row per output pixel,
// K = 9 C.  The kernels' parameters carry the same geometry fields.
template <class P>
inline int set_conv3x3(const char* fn, P& p, const float* in, int batch, int H, int W, int C, int stride,
                       int c_multiple) {
    O3DML_CHECK(in && batch > 0 && H > 0 && W > 0, "%s: bad input", fn);
    O3DML_CHECK((C % c_multiple) == 0, "%s: input channels must be a multiple of %d", fn, c_multiple);
    O3DML_CHECK(stride == 1 || stride == 2, "%s: stride 1 or 2", fn);
    O3DML_CHECK((reinterpret_cast<uintptr_t>(in) & 15) == 0, "%s: input must be 16-byte aligned", fn);
    p.mode = 1;
    p.nsrc = 1;
    p.src[0].data = in;
    p.H = H; p.W = W; p.C = C; p.stride = stride;
    p.OH = (H + 2 - 3) / stride + 1;
    p.OW = (W + 2 - 3) / stride + 1;
    p.N = (int64_t)batch * p.OH * p.OW;
    p.K = 9 * C;
    return O3DML_OK;
}

// A transposed convolution with kernel == stride over an NHWC input is a 1x1 product over the input pixels (one
// identity source of C channels, stride^2 * out_channels columns) whose output is pixel-shuffled.  scale / shift come
// tiled to [stride^2 * out_channels].
template <class P>
inline int set_deconv(const char* fn, P& p, const void* weight, const float* in, int batch, int H, int W, int C,
                      int stride, const float* scale, const float* shift, int act, float slope, float* out, int out_ld,
                      int out_channels) {
    O3DML_CHECK(in && batch > 0 && H > 0 && W > 0 && stride >= 1, "%s: bad input", fn);
    o3dml_src_t s = {};
    s.data = in;
    s.rows = (int64_t)batch * H * W;
    s.channels = C;
    s.ld = C;
    p.mode = 0;
    p.nsrc = 1;
    p.N = s.rows;
    int rc = set_srcs(fn, &s, 1, p.src, p.koff);
    if (rc) return rc;
    p.K = C;
    rc = set_epilogue(fn, p, weight, scale, shift, nullptr, 0, act, slope, out, out_ld, stride * stride * out_channels,
                      0);
    if (rc) return rc;
    p.ep.mode = 2;
    p.ep.ds = stride; p.ep.dIH = H; p.ep.dIW = W; p.ep.dC = out_channels;
    return O3DML_OK;
}

}  // namespace o3dml
