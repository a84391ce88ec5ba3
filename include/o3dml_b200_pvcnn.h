/* o3dml_b200_pvcnn.h -- the PVCNN entries of the C ABI of libo3dml_b200.so: voxel coordinates and cells, the mean of
 * the points of every cell, the 3x3x3 tensor-core convolution and trilinear devoxelization.  Conventions (status
 * return, o3dml_last_error, device pointers, the stream argument, O3DML_ABI_VERSION) are those of o3dml_b200.h, which
 * this header includes.  Every entry enqueues at least one kernel and takes no workspace: scratch comes as typed
 * output arguments whose size follows from the shapes.  open3d_ml_b200._lib.PVCNN_EXPORTS binds exactly what is
 * declared here (tests/test_abi_pvcnn.py). */
#ifndef O3DML_B200_PVCNN_H
#define O3DML_B200_PVCNN_H
#include "o3dml_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Grids of PVConv (pvcnn.py:559-664) are channels-last: [batch, X, Y, Z, C] with z fastest among the spatial axes, so
 * cell (x, y, z) of cloud b is row b * r^3 + (x * r + y) * r + z.
 *
 * Voxelization coordinates (pvcnn.py:642-664, normalize = True).  coords [batch * num_points, 3] point rows.  Per
 * cloud, the mean of its points and denom = 2 * max_n |c_n - mean| + eps are reduced in a fixed order and written to
 * stats [batch, 4]; per point voxel_coords [batch * num_points, 3] = clamp(((c - mean) / denom + 0.5) * r, 0, r - 1),
 * the coordinates trilinear devoxelization interpolates at, and cell_ids int32 [batch * num_points] = the row of the
 * cell (round half to even per axis) the point is averaged into.  batch * r^3 < 2^31.  Two kernels, no host read. */
O3DML_API int o3dml_pv_voxel_cells(const float* coords, int batch, int num_points, int resolution, float eps,
                                   float* stats, float* voxel_coords, int32_t* cell_ids, void* stream);

/* avg_voxelize (pvcnn.py:579-619) from the points grouped by cell: cell_row_splits int64 [num_cells + 1] and point_ids
 * int32, as o3dml_invert_neighbors_list gives them for one cell id per point.  grid [num_cells, channels_pad]: the mean
 * of features [., features_ld] over the points of the cell, added in list order; zeros for an empty cell and in
 * channels [channels, channels_pad).  Every element of grid is written. */
O3DML_API int o3dml_pv_cell_mean(const int64_t* cell_row_splits, const int32_t* point_ids, int64_t num_cells,
                                 const float* features, int features_ld, int channels, int channels_pad, float* grid,
                                 void* stream);

/* Conv3d(kernel 3, padding 1, stride 1) over a channels-last grid on the tensor cores (3xTF32, as o3dml_conv3x3_nhwc_tc):
 * in [batch, X, Y, Z, C], C % 32 == 0, out [batch, X, Y, Z, out_channels]; weight image of the [27 C, out_channels]
 * matrix whose row is ((kx * 3 + ky) * 3 + kz) * C + c. */
O3DML_API int o3dml_conv3x3x3_ndhwc_tc(const float* in, int batch, int X, int Y, int Z, int C, const void* weight_image,
                                       int k_pad, int n_pad, const float* scale, const float* shift, int act,
                                       float slope, float* out, int out_channels, void* stream);

/* open3d.ml.torch.ops.trilinear_devoxelize_forward on a channels-last grid [batch * r^3, grid_ld] at voxel_coords
 * [batch * num_points, 3] in [0, r - 1].  Per axis lo = floor(v), d = v - lo, hi = lo + (d > 0 ? 1 : 0); corner k =
 * 0..7 takes hi on x / y / z where bit 2 / 1 / 0 of k is set, its weight is the product of d (hi) or 1 - d (lo) and its
 * cell is (x * r + y) * r + z.  out [batch * num_points, out_ld] gets (accumulate = 0) or is increased by
 * (accumulate = 1) the weighted sum of the eight rows, added in corner order.  inds int32 / wgts float
 * [batch, 8, num_points] are written when not null. */
O3DML_API int o3dml_trilinear_devoxelize(const float* voxel_coords, int batch, int num_points, int resolution,
                                         const float* grid, int channels, int grid_ld, int accumulate, float* out,
                                         int out_ld, int32_t* inds, float* wgts, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3DML_B200_PVCNN_H */
