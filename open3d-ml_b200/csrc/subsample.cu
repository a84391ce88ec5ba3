// subsample.cu -- grid subsampling (barycentre per voxel), the reduction half of
//   open3d.ml.contrib.subsample        ml3d/datasets/utils/dataprocessing.py:14-49
//   open3d.ml.contrib.subsample_batch  ml3d/torch/models/kpconv.py:2037-2164 (batch_grid_subsampling)
// and of open3d.ml.torch.ops.voxel_pooling (north-star op surface, no call site in the reference).
// The partition half is o3dml_voxelize (hash -> stable radix sort -> segment): this kernel consumes
// its CSR voxel lists (voxel_point_row_splits + voxel_point_indices, point ids ascending inside a
// voxel) and writes, per voxel, the mean position, the mean of every feature channel and the most
// frequent label (ties -> the smallest label).  Sums run sequentially in ascending point-id order in
// fp32 (no FMA, one rounding per add, then one division), so the result is bit-reproducible against
// oracle/ops_ref.c oracle_voxel_reduce.  HBM-bound: (12 + 4F + 4) B per point in, (12 + 4F + 4) B per
// voxel out.
#include "../../include/o3dml_b200.h"
#include "common.cuh"

namespace o3dml {

// one thread per (voxel, channel): channels [0,3) = xyz, [3, 3+F) = features; feature_mode 1 = max
__global__ void voxel_reduce_kernel(const float* __restrict__ pts, int pld, const float* __restrict__ feat, int F,
                                    int fld, const int64_t* __restrict__ vrs, const int64_t* __restrict__ pidx,
                                    const int64_t* __restrict__ d_num_voxels, int64_t bound, int position_mode,
                                    int feature_mode, float* __restrict__ out_pts, float* __restrict__ out_feat) {
    const int C = 3 + F;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t v = t / C;
    const int c = (int)(t - v * C);
    const int64_t M = d_num_voxels ? min(*d_num_voxels, bound) : bound;
    if (v >= M) return;
    const int64_t s = vrs[v], e = vrs[v + 1];
    const bool is_pos = c < 3;
    if (is_pos && !out_pts) return;
    if (!is_pos && !out_feat) return;
    const float* src = is_pos ? pts + c : feat + (c - 3);
    const int ld = is_pos ? pld : fld;
    const int mode = is_pos ? position_mode : feature_mode;   // 0 mean, 1 max, 2 first (nearest_neighbor stand-in)
    float acc = mode == 1 ? -INFINITY : 0.f;
    for (int64_t j = s; j < e; ++j) {
        const float x = src[(size_t)pidx[j] * ld];
        if (mode == 0) acc = __fadd_rn(acc, x);
        else if (mode == 1) acc = (x > acc || x != x) ? x : acc;  // a NaN stays (fmaxf would drop it)
        else if (j == s) acc = x;
    }
    if (mode == 0) acc = __fdiv_rn(acc, (float)(e - s));
    if (is_pos) out_pts[(size_t)v * 3 + c] = acc;
    else out_feat[(size_t)v * F + (c - 3)] = acc;
}

// one thread per voxel: most frequent label, ties -> smallest label
__global__ void voxel_label_kernel(const int32_t* __restrict__ labels, const int64_t* __restrict__ vrs,
                                   const int64_t* __restrict__ pidx, const int64_t* __restrict__ d_num_voxels,
                                   int64_t bound, int32_t* __restrict__ out_labels) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t M = d_num_voxels ? min(*d_num_voxels, bound) : bound;
    if (v >= M) return;
    const int64_t s = vrs[v], e = vrs[v + 1];
    int32_t best = 0;
    int64_t best_n = 0;
    for (int64_t i = s; i < e; ++i) {
        const int32_t l = labels[pidx[i]];
        bool seen = false;
        for (int64_t j = s; j < i && !seen; ++j) seen = labels[pidx[j]] == l;
        if (seen) continue;
        int64_t n = 1;
        for (int64_t j = i + 1; j < e; ++j) n += labels[pidx[j]] == l;
        if (n > best_n || (n == best_n && l < best)) { best = l; best_n = n; }
    }
    out_labels[v] = best;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_voxel_reduce(const float* points, int point_stride, const float* features, int feat_channels,
                                  int feat_stride, const int32_t* labels, const int64_t* voxel_row_splits,
                                  const int64_t* voxel_point_indices, const int64_t* d_num_voxels,
                                  int64_t num_voxels_bound, int position_mode, int feature_mode, float* out_points,
                                  float* out_features, int32_t* out_labels, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(points && voxel_row_splits && voxel_point_indices, "voxel_reduce: null input");
    O3DML_CHECK(point_stride >= 3 && feat_channels >= 0, "voxel_reduce: bad strides");
    O3DML_CHECK(position_mode >= 0 && position_mode <= 2 && feature_mode >= 0 && feature_mode <= 2,
                "voxel_reduce: modes are 0 (mean), 1 (max), 2 (first)");
    O3DML_CHECK(feat_channels == 0 || (features && out_features && feat_stride >= feat_channels),
                "voxel_reduce: features need an output and a stride");
    O3DML_CHECK(!labels || out_labels, "voxel_reduce: labels need an output");
    if (num_voxels_bound <= 0) return O3DML_OK;
    const int C = 3 + feat_channels;
    const int64_t total = num_voxels_bound * C;
    O3DML_CUDA(launch<voxel_reduce_kernel>((unsigned)ceil_div<int64_t>(total, 256), 256, 0, st, points, point_stride,
                                           features, feat_channels, feat_stride, voxel_row_splits, voxel_point_indices,
                                           d_num_voxels, num_voxels_bound, position_mode, feature_mode, out_points,
                                           out_features));
    if (labels)
        O3DML_CUDA(launch<voxel_label_kernel>((unsigned)ceil_div<int64_t>(num_voxels_bound, 128), 128, 0, st, labels,
                                              voxel_row_splits, voxel_point_indices, d_num_voxels, num_voxels_bound,
                                              out_labels));
    return O3DML_OK;
}

// ---- open3d.ml.torch.ops.reduce_subarrays_sum(values, row_splits) ---------------------------------
//   call site: ml3d/torch/models/sparseconvnet.py:318-324 (per-voxel feature sums of InputLayer).
// out[i] = sum of values[row_splits[i] : row_splits[i+1]], sequential fp32 adds in index order (one thread per
// segment: deterministic and bit-equal to the oracle; segments are voxels, i.e. short).
namespace o3dml {
__global__ void reduce_subarrays_kernel(const float* __restrict__ values, const int64_t* __restrict__ splits, int64_t rows,
                                        float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    float acc = 0.f;
    for (int64_t j = splits[i]; j < splits[i + 1]; ++j) acc = __fadd_rn(acc, values[j]);
    out[i] = acc;
}
}  // namespace o3dml

extern "C" int o3dml_reduce_subarrays_sum(const float* values, const int64_t* row_splits, int64_t num_rows, float* out,
                                          void* stream) {
    if (num_rows <= 0) return O3DML_OK;
    O3DML_CHECK(values && row_splits && out, "reduce_subarrays_sum: null input");
    O3DML_CUDA(launch<reduce_subarrays_kernel>((unsigned)ceil_div<int64_t>(num_rows, 256), 256, 0, (cudaStream_t)stream,
                                               values, row_splits, num_rows, out));
    return O3DML_OK;
}
