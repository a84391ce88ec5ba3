// cconv.cu -- open3d.ml.torch.ops.continuous_conv (north-star op surface; no call site in the reference tree,
// README.md:91 lists it).  Contract (upstream Open3D absent: parity unpinned; oracle/ops_ref.c oracle_continuous_conv):
//   for output o with neighbours n in [row_splits[o], row_splits[o+1]):
//     p  = (inp_pos[n] - out_pos[o]) * 2 / extent + offset          relative position, ball of diameter `extent` -> [-1, 1]^3
//     p' = coordinate_mapping(p)      identity | ball_to_cube_radial: p * |p|_2 / |p|_inf (0 at the centre)
//     u_a = align_corners ? (p'_a + 1) / 2 * (S_a - 1) : (p'_a + 1) / 2 * S_a - 0.5      a = x, y, z; S = filter size
//     W(u) = nearest | trilinear (indices clamped to the border: "linear") | trilinear, zero outside ("linear_border")
//     out[o] += importance[n] * W(u)^T f[n];   normalize: divide by sum of importance (or the neighbour count)
//   filters [Sz, Sy, Sx, Cin, Cout].
// open3d.ml.torch.ops.continuous_conv_transpose, the exact adjoint of the op above (float64 oracle:
//   tests/cconv_transpose_oracle.py):
//   for output o with neighbours n (inputs) in [row_splits[o], row_splits[o+1]):
//     p  = (out_pos[o] - inp_pos[n]) * 2 / extent_n + offset         the input is the centre; extent indexed by n
//     out[o] = oimp[o] * sum_n importance[n] * s_n * W(u)^T f[n]      s_n = 1 / inp_neighbors_importance_sum[n], or
//                                                                     1 / (n's forward neighbour count); 1 without
//                                                                     normalize or for a zero divisor
//   Same mapping, interpolation and filter layout; TRANSPOSE selects it at compile time.
// invert_neighbors_list: the ragged lists (row i -> ids j) regrouped by id (row j -> rows i), by a stable radix sort.
// One CTA per output point, threads over output channels (coalesced filter rows), neighbour features staged in
// shared memory; FP32 SIMT (the per-neighbour filter is interpolated, not a dense contraction over a shared operand).
#include "../../include/o3dml_b200.h"
#include "common.cuh"
#include "prims.cuh"

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
    // transposed op only (appended, so that the forward's parameter offsets stay as they were)
    const float* out_importance;      // [num_out] or NULL
    const float* inp_imp_sum;         // [num_inp] or NULL: the normaliser of input n
    const int64_t* inp_row_splits;    // [num_inp + 1] or NULL: the forward lists, whose lengths normalise otherwise
    float Sf[3];                      // S as floats: the bounds of cconv_corners' clamps, read from the parameters
};

// s_n of the transposed op: the forward's normaliser of input n, inverted (1 for a zero divisor or without normalize)
__device__ __forceinline__ float cconv_inp_scale(const CConvParams& p, int64_t n) {
    if (!p.normalize) return 1.f;
    const float d = p.inp_imp_sum ? p.inp_imp_sum[n] : (float)(p.inp_row_splits[n + 1] - p.inp_row_splits[n]);
    return d != 0.f ? 1.f / d : 1.f;
}

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
    // A far neighbour's floor(u) can be past the int range, so it is clamped in float before it becomes an int: to
    // the filter for nearest, to [-2, S] for the linear kinds (both corners outside on either side stay outside).
    // fmaxf takes a NaN floor to the low end: cell 0 for nearest; both corners outside for the linear kinds, which
    // linear_border weighs 0 and linear with the NaN weight of the unclamped floor, as the oracle does.
    if (p.interpolation == 0) {
        int c[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) c[a] = (int)fminf(fmaxf(floorf(u[a] + 0.5f), 0.f), p.Sf[a] - 1.f);
        idx[0] = (c[2] * p.S[1] + c[1]) * p.S[0] + c[0];
        wgt[0] = 1.f;
        return 1;
    }
    int i0[3];
    float f[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float fl = floorf(u[a]);
        i0[a] = (int)fminf(fmaxf(fl, -2.f), p.Sf[a]);
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

template <bool TRANSPOSE>
__global__ void __launch_bounds__(128) cconv_kernel(const CConvParams p) {
    extern __shared__ float sf[];      // [cin] features of the current neighbour
    const int64_t o = blockIdx.x;
    const int64_t s = p.row_splits[o], e = p.row_splits[o + 1];
    float inv = 0.f;                   // transposed: the extent belongs to the neighbour and is read per entry
    if constexpr (!TRANSPOSE) {
        const float ext = p.extents[p.extents_per_point ? o : 0];
        inv = ext > 0.f ? 2.0f / ext : 0.f;
    }
    constexpr int MAXCO = 8;           // output channels per thread: cout <= 1024
    float acc[MAXCO];
#pragma unroll
    for (int i = 0; i < MAXCO; ++i) acc[i] = 0.f;
    float norm = 0.f;
    for (int64_t j = s; j < e; ++j) {
        const int64_t n = load_index(p.nbr_index, j, p.nbr_is64);
        float imp = p.nbr_importance ? p.nbr_importance[j] : 1.f;
        if constexpr (TRANSPOSE) {
            imp *= cconv_inp_scale(p, n);
            const float ext = p.extents[p.extents_per_point ? n : 0];
            inv = ext > 0.f ? 2.0f / ext : 0.f;
        } else {
            if (p.inp_importance) imp *= p.inp_importance[n];
            norm += imp;
        }
        __syncthreads();
        for (int c = threadIdx.x; c < p.cin; c += blockDim.x) sf[c] = p.inp_feat[(size_t)n * p.cin + c] * imp;
        __syncthreads();
        float rel[3];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            rel[a] = (TRANSPOSE ? p.out_pos[3 * o + a] - p.inp_pos[3 * n + a] : p.inp_pos[3 * n + a] - p.out_pos[3 * o + a]) *
                         inv + p.offset[a];
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
    float scale;
    if constexpr (TRANSPOSE)
        scale = p.out_importance ? p.out_importance[o] : 1.f;
    else
        scale = (p.normalize && norm != 0.f) ? 1.f / norm : 1.f;
#pragma unroll
    for (int i = 0; i < MAXCO; ++i) {
        const int co = threadIdx.x + i * 128;
        if (co < p.cout) p.out[(size_t)o * p.cout + co] = acc[i] * scale;
    }
}

// The checks both directions share, then one CTA per output.  `importance` is inp_importance of the forward op and
// out_importance of the transposed one; inp_imp_sum / inp_row_splits are read by the transposed op only.
template <bool TRANSPOSE>
static int cconv_run(const char* op, const float* filters, int size_x, int size_y, int size_z, int in_channels,
                     int out_channels, const float* out_positions, int64_t num_out, const float* extents,
                     int extents_per_point, const float* h_offset, const float* inp_positions,
                     const float* inp_features, int64_t num_inp, const float* importance, const float* inp_imp_sum,
                     const int64_t* inp_row_splits, const void* neighbors_index, int index_is64,
                     const float* neighbors_importance, const int64_t* neighbors_row_splits, int align_corners,
                     int coordinate_mapping, int normalize, int interpolation, float* out, cudaStream_t st) {
    O3DML_CHECK(size_x >= 1 && size_y >= 1 && size_z >= 1 && in_channels >= 1 && out_channels >= 1 && out_channels <= 1024,
                "%s: bad filter shape (out_channels <= 1024)", op);
    // one input row is staged in the 48 KB of dynamic shared memory a kernel gets without opting in
    O3DML_CHECK(in_channels <= 48 * 1024 / (int)sizeof(float), "%s: in_channels must be <= 12288", op);
    O3DML_CHECK(coordinate_mapping == 0 || coordinate_mapping == 1,
                "%s: coordinate_mapping must be identity (0) or ball_to_cube_radial (1)", op);
    O3DML_CHECK(interpolation >= 0 && interpolation <= 2, "%s: interpolation 0 nearest, 1 linear, 2 linear_border", op);
    O3DML_CHECK(!TRANSPOSE || !normalize || inp_imp_sum || inp_row_splits,
                "%s: normalize needs inp_neighbors_importance_sum or inp_neighbors_row_splits", op);
    if (num_out <= 0) return O3DML_OK;
    CConvParams p;
    p.filters = filters;
    p.S[0] = size_x; p.S[1] = size_y; p.S[2] = size_z;
    for (int a = 0; a < 3; ++a) p.Sf[a] = (float)p.S[a];
    p.cin = in_channels; p.cout = out_channels;
    p.out_pos = out_positions; p.inp_pos = inp_positions; p.inp_feat = inp_features;
    p.inp_importance = TRANSPOSE ? nullptr : importance;
    p.nbr_index = neighbors_index; p.nbr_is64 = index_is64; p.nbr_importance = neighbors_importance;
    p.row_splits = neighbors_row_splits; p.extents = extents; p.extents_per_point = extents_per_point;
    for (int a = 0; a < 3; ++a) p.offset[a] = h_offset ? h_offset[a] : 0.f;
    p.align_corners = align_corners; p.mapping = coordinate_mapping; p.interpolation = interpolation;
    p.normalize = normalize; p.num_out = num_out; p.num_inp = num_inp; p.out = out;
    p.out_importance = TRANSPOSE ? importance : nullptr;
    p.inp_imp_sum = inp_imp_sum; p.inp_row_splits = inp_row_splits;
    O3DML_CUDA(launch<cconv_kernel<TRANSPOSE>>((unsigned)num_out, 128, (size_t)in_channels * sizeof(float), st, p));
    return O3DML_OK;
}

// ------------------------------------------------------------------------------------------ invert_neighbors_list
// Sort key of entry e: its id, or num_points when the id is out of range (those sort after every row and are dropped).
__global__ void __launch_bounds__(256) inv_keys_kernel(const void* __restrict__ index, int is64, int64_t num_entries,
                                                        int64_t num_points, uint64_t* __restrict__ keys) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= num_entries) return;
    const int64_t id = load_index(index, e, is64);
    keys[e] = (uint64_t)(id >= 0 && id < num_points ? id : num_points);
}

// row_splits[r] = the number of sorted keys below r (a lower bound per row): empty rows need no special case and
// row_splits[num_points] is the number of entries kept.
__global__ void __launch_bounds__(256) inv_splits_kernel(const uint64_t* __restrict__ keys, int64_t num_entries,
                                                          int64_t num_points, int64_t* __restrict__ row_splits) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > num_points) return;
    int64_t lo = 0, hi = num_entries;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < (uint64_t)r) lo = mid + 1; else hi = mid;
    }
    row_splits[r] = lo;
}

// Sorted position t holds entry perm[t] = vals[t]; its source row is the input row whose range holds that entry.
__global__ void __launch_bounds__(256) inv_emit_kernel(const uint32_t* __restrict__ vals, int64_t num_entries,
                                                        const int64_t* __restrict__ inp_row_splits, int64_t num_inp,
                                                        void* __restrict__ out_index, int is64,
                                                        int64_t* __restrict__ permutation) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= num_entries) return;
    const int64_t e = vals[t];
    int64_t lo = 0, hi = num_inp;      // the last row i with inp_row_splits[i] <= e
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (inp_row_splits[mid] <= e) lo = mid; else hi = mid - 1;
    }
    if (is64) ((int64_t*)out_index)[t] = lo;
    else ((int32_t*)out_index)[t] = (int32_t)lo;
    permutation[t] = e;
}

static RadixSortBufs inv_carve(Workspace& ws, int64_t num_entries) {
    return radix_sort_carve(ws, num_entries);
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
    O3DML_CHECK(num_out >= 0 && num_inp >= 0, "continuous_conv: negative size");
    O3DML_CHECK(filters && extents && neighbors_row_splits && (num_out == 0 || (out_positions && out)) &&
                    (num_inp == 0 || (inp_positions && inp_features)),
                "continuous_conv: null input");
    return cconv_run<false>("continuous_conv", filters, size_x, size_y, size_z, in_channels, out_channels, out_positions,
                            num_out, extents, extents_per_point, h_offset, inp_positions, inp_features, num_inp,
                            inp_importance, nullptr, nullptr, neighbors_index, index_is64, neighbors_importance,
                            neighbors_row_splits, align_corners, coordinate_mapping, normalize, interpolation, out,
                            (cudaStream_t)stream);
}

extern "C" int o3dml_continuous_conv_transpose(const float* filters, int size_x, int size_y, int size_z,
                                               int in_channels, int out_channels, const float* out_positions,
                                               int64_t num_out, const float* out_importance, const float* extents,
                                               int extents_per_point, const float* h_offset,
                                               const float* inp_positions, const float* inp_features, int64_t num_inp,
                                               const float* inp_neighbors_importance_sum,
                                               const int64_t* inp_neighbors_row_splits, const void* neighbors_index,
                                               int index_is64, const float* neighbors_importance,
                                               const int64_t* neighbors_row_splits, int align_corners,
                                               int coordinate_mapping, int normalize, int interpolation, float* out,
                                               void* stream) {
    O3DML_CHECK(num_out >= 0 && num_inp >= 0, "continuous_conv_transpose: negative size");
    O3DML_CHECK(filters && extents && neighbors_row_splits && (num_out == 0 || (out_positions && out)) &&
                    (num_inp == 0 || (inp_positions && inp_features)),
                "continuous_conv_transpose: null input");
    return cconv_run<true>("continuous_conv_transpose", filters, size_x, size_y, size_z, in_channels, out_channels,
                           out_positions, num_out, extents, extents_per_point, h_offset, inp_positions, inp_features,
                           num_inp, out_importance, inp_neighbors_importance_sum, inp_neighbors_row_splits,
                           neighbors_index, index_is64, neighbors_importance, neighbors_row_splits, align_corners,
                           coordinate_mapping, normalize, interpolation, out, (cudaStream_t)stream);
}

extern "C" size_t o3dml_invert_neighbors_list_workspace_bytes(int64_t num_entries) {
    return Workspace::measure(inv_carve, num_entries);
}

extern "C" int o3dml_invert_neighbors_list(int64_t num_points, const void* inp_neighbors_index, int index_is64,
                                           const int64_t* inp_neighbors_row_splits, int64_t num_inp,
                                           int64_t num_entries, void* neighbors_index, int64_t* neighbors_row_splits,
                                           int64_t* permutation, void* workspace, size_t workspace_bytes,
                                           void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(num_points >= 0 && num_inp >= 0 && num_entries >= 0, "invert_neighbors_list: negative size");
    // the sort carries entry ids as uint32 values
    O3DML_CHECK(num_entries < ((int64_t)1 << 32), "invert_neighbors_list: 2^32 or more entries");
    O3DML_CHECK(index_is64 || num_inp <= INT32_MAX, "invert_neighbors_list: more than 2^31 - 1 rows for int32 indices");
    O3DML_CHECK(neighbors_row_splits && (num_entries == 0 || (inp_neighbors_index && inp_neighbors_row_splits &&
                                                               neighbors_index && permutation)),
                "invert_neighbors_list: null input");
    Workspace ws(workspace, workspace_bytes);
    RadixSortBufs b = inv_carve(ws, num_entries);
    O3DML_CHECK_WORKSPACE(ws, "invert_neighbors_list");

    int num_bits = 1;      // the largest key is num_points
    while (num_bits < 64 && ((uint64_t)num_points >> num_bits) != 0) ++num_bits;
    const int T = 256;
    const unsigned nb = (unsigned)ceil_div<int64_t>(num_entries, T);
    if (num_entries > 0) {
        O3DML_CUDA(launch<inv_keys_kernel>(nb, T, 0, st, inp_neighbors_index, index_is64, num_entries, num_points,
                                           b.keys_a));
        O3DML_CUDA(radix_sort_pairs(b, true, num_entries, num_bits, st));
    }
    O3DML_CUDA(launch<inv_splits_kernel>((unsigned)ceil_div<int64_t>(num_points + 1, T), T, 0, st, b.keys_a,
                                         num_entries, num_points, neighbors_row_splits));
    if (num_entries > 0)
        O3DML_CUDA(launch<inv_emit_kernel>(nb, T, 0, st, b.vals_a, num_entries, inp_neighbors_row_splits, num_inp,
                                           neighbors_index, index_is64, permutation));
    return O3DML_OK;
}
