// cconv.cu -- open3d.ml.torch.ops.continuous_conv (north-star op surface; no call site in the reference tree,
// README.md:91 lists it).  Contract (upstream Open3D absent: parity unpinned; oracle/ops_ref.c oracle_continuous_conv):
//   for output o with neighbours n in [row_splits[o], row_splits[o+1]):
//     p  = (inp_pos[n] - out_pos[o]) * 2 / extent + offset          relative position, ball of diameter `extent` -> [-1, 1]^3
//     p' = coordinate_mapping(p)      identity | ball_to_cube_radial: p * |p|_2 / |p|_inf (0 at the centre)
//     u_a = align_corners ? (p'_a + 1) / 2 * (S_a - 1) : (p'_a + 1) / 2 * S_a - 0.5      a = x, y, z; S = filter size
//     W(u) = nearest | trilinear (indices clamped to the border: "linear") | trilinear, zero outside ("linear_border")
//     out[o] += importance[n] * W(u)^T f[n];   normalize: divide by sum of importance (or the neighbour count)
//   filters [Sz, Sy, Sx, Cin, Cout].
// One CTA per output point, threads over output channels (coalesced filter rows), neighbour features staged in
// shared memory; FP32 SIMT (the per-neighbour filter is interpolated, not a dense contraction over a shared operand).
#include "../../include/o3dml_b200.h"
#include "common.cuh"

namespace o3dml {

struct CConvParams {
    const float* filters;
    int S[3];             // Sx, Sy, Sz
    int cin, cout;
    const float* out_pos;
    const float* inp_pos;
    const float* inp_feat;
    const float* inp_importance;      // may be NULL
    const void* nbr_index;
    int nbr_is64;
    const float* nbr_importance;      // may be NULL
    const int64_t* row_splits;
    const float* extents;             // [1] or [num_out]
    int extents_per_point;
    float offset[3];
    int align_corners, mapping, interpolation, normalize;   // mapping 0 identity, 1 ball_to_cube_radial; interp 0 nn, 1 linear, 2 linear_border
    int64_t num_out, num_inp;
    float* out;
};

__device__ __forceinline__ int cconv_corners(const CConvParams& p, const float* rel, int* idx, float* wgt) {
    float q[3] = {rel[0], rel[1], rel[2]};
    if (p.mapping == 1) {
        const float n2 = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        const float ni = fmaxf(fabsf(q[0]), fmaxf(fabsf(q[1]), fabsf(q[2])));
        const float s = ni > 0.f ? n2 / ni : 0.f;
        q[0] *= s; q[1] *= s; q[2] *= s;
    }
    float u[3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
        u[a] = p.align_corners ? (q[a] + 1.f) * 0.5f * (float)(p.S[a] - 1) : (q[a] + 1.f) * 0.5f * (float)p.S[a] - 0.5f;
    if (p.interpolation == 0) {
        int c[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) c[a] = min(max((int)floorf(u[a] + 0.5f), 0), p.S[a] - 1);
        idx[0] = (c[2] * p.S[1] + c[1]) * p.S[0] + c[0];
        wgt[0] = 1.f;
        return 1;
    }
    int i0[3];
    float f[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float fl = floorf(u[a]);
        i0[a] = (int)fl;
        f[a] = u[a] - fl;
    }
    int n = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        int ii[3];
        float w = 1.f;
        bool inside = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int bit = (c >> a) & 1;
            int i = i0[a] + bit;
            w *= bit ? f[a] : 1.f - f[a];
            if (i < 0 || i >= p.S[a]) {
                inside = false;
                i = min(max(i, 0), p.S[a] - 1);
            }
            ii[a] = i;
        }
        if (p.interpolation == 2 && !inside) w = 0.f;
        idx[n] = (ii[2] * p.S[1] + ii[1]) * p.S[0] + ii[0];
        wgt[n] = w;
        ++n;
    }
    return n;
}

__global__ void __launch_bounds__(128) cconv_kernel(const CConvParams p) {
    extern __shared__ float sf[];      // [cin] features of the current neighbour
    const int64_t o = blockIdx.x;
    const int64_t s = p.row_splits[o], e = p.row_splits[o + 1];
    const float ext = p.extents[p.extents_per_point ? o : 0];
    const float inv = ext > 0.f ? 2.0f / ext : 0.f;
    constexpr int MAXCO = 8;           // output channels per thread: cout <= 1024
    float acc[MAXCO];
#pragma unroll
    for (int i = 0; i < MAXCO; ++i) acc[i] = 0.f;
    float norm = 0.f;
    for (int64_t j = s; j < e; ++j) {
        const int64_t n = load_index(p.nbr_index, j, p.nbr_is64);
        float imp = p.nbr_importance ? p.nbr_importance[j] : 1.f;
        if (p.inp_importance) imp *= p.inp_importance[n];
        norm += imp;
        __syncthreads();
        for (int c = threadIdx.x; c < p.cin; c += blockDim.x) sf[c] = p.inp_feat[(size_t)n * p.cin + c] * imp;
        __syncthreads();
        float rel[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) rel[a] = (p.inp_pos[3 * n + a] - p.out_pos[3 * o + a]) * inv + p.offset[a];
        int idx[8];
        float wgt[8];
        const int nc = cconv_corners(p, rel, idx, wgt);
        for (int k = 0; k < nc; ++k) {
            if (wgt[k] == 0.f) continue;
            const float* w = p.filters + (size_t)idx[k] * p.cin * p.cout;
            for (int ci = 0; ci < p.cin; ++ci) {
                const float fv = sf[ci] * wgt[k];
#pragma unroll
                for (int i = 0; i < MAXCO; ++i) {
                    const int co = threadIdx.x + i * 128;
                    if (co < p.cout) acc[i] = fmaf(fv, w[(size_t)ci * p.cout + co], acc[i]);
                }
            }
        }
    }
    const float scale = (p.normalize && norm != 0.f) ? 1.f / norm : 1.f;
#pragma unroll
    for (int i = 0; i < MAXCO; ++i) {
        const int co = threadIdx.x + i * 128;
        if (co < p.cout) p.out[(size_t)o * p.cout + co] = acc[i] * scale;
    }
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_continuous_conv(const float* filters, int size_x, int size_y, int size_z, int in_channels,
                                     int out_channels, const float* out_positions, int64_t num_out,
                                     const float* extents, int extents_per_point, const float* h_offset,
                                     const float* inp_positions, const float* inp_features, int64_t num_inp,
                                     const float* inp_importance, const void* neighbors_index, int index_is64,
                                     const float* neighbors_importance, const int64_t* neighbors_row_splits,
                                     int align_corners, int coordinate_mapping, int normalize, int interpolation,
                                     float* out, void* stream) {
    O3DML_CHECK(filters && out_positions && extents && inp_positions && inp_features && neighbors_row_splits && out,
                "continuous_conv: null input");
    O3DML_CHECK(size_x >= 1 && size_y >= 1 && size_z >= 1 && in_channels >= 1 && out_channels >= 1 && out_channels <= 1024,
                "continuous_conv: bad filter shape (out_channels <= 1024)");
    // one input row is staged in the 48 KB of dynamic shared memory a kernel gets without opting in
    O3DML_CHECK(in_channels <= 48 * 1024 / (int)sizeof(float), "continuous_conv: in_channels must be <= 12288");
    O3DML_CHECK(coordinate_mapping == 0 || coordinate_mapping == 1,
                "continuous_conv: coordinate_mapping must be identity (0) or ball_to_cube_radial (1)");
    O3DML_CHECK(interpolation >= 0 && interpolation <= 2, "continuous_conv: interpolation 0 nearest, 1 linear, 2 linear_border");
    if (num_out <= 0) return O3DML_OK;
    CConvParams p;
    p.filters = filters;
    p.S[0] = size_x; p.S[1] = size_y; p.S[2] = size_z;
    p.cin = in_channels; p.cout = out_channels;
    p.out_pos = out_positions; p.inp_pos = inp_positions; p.inp_feat = inp_features; p.inp_importance = inp_importance;
    p.nbr_index = neighbors_index; p.nbr_is64 = index_is64; p.nbr_importance = neighbors_importance;
    p.row_splits = neighbors_row_splits; p.extents = extents; p.extents_per_point = extents_per_point;
    for (int a = 0; a < 3; ++a) p.offset[a] = h_offset ? h_offset[a] : 0.f;
    p.align_corners = align_corners; p.mapping = coordinate_mapping; p.interpolation = interpolation;
    p.normalize = normalize; p.num_out = num_out; p.num_inp = num_inp; p.out = out;
    O3DML_CUDA(launch<cconv_kernel>((unsigned)num_out, 128, (size_t)in_channels * sizeof(float), (cudaStream_t)stream, p));
    return O3DML_OK;
}
