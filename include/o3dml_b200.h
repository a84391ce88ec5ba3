/*
 * o3dml_b200.h -- C ABI of libo3dml_b200.so: Hopper (sm_90a) point-cloud operators
 * that drop in behind the `open3d.ml.torch.{ops,layers}` / `open3d.core.nns` surface
 * consumed by isl-org/Open3D-ML's PyTorch models, plus the fused per-model hot layers.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless its name starts with h_ (host);
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, no
 *     function synchronises the device or allocates memory;
 *   - scratch memory comes from the caller (`workspace`, sized by the matching
 *     *_workspace_bytes function, which returns exactly the bytes the entry uses);
 *     an entry given too small a workspace returns 2 before it enqueues anything,
 *     and o3dml_last_error() names the bytes it needed; outputs are
 *     caller-allocated, inputs are never written or retained;
 *   - return value 0 = success; otherwise o3dml_last_error() describes the failure
 *     (the Python layer raises RuntimeError, as TORCH_CHECK does upstream);
 *   - data-dependent output sizes are reported through small device counters
 *     (`d_*`) so that the caller decides when to pay the device->host read.
 *
 * Each entry point names the reference interface it replaces
 * (file:line under /root/reference, SURVEY.md section 8a/8b).
 */
#ifndef O3DML_B200_H
#define O3DML_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define O3DML_ABI_VERSION 2
#define O3DML_API __attribute__((visibility("default")))

/* activation codes */
#define O3DML_ACT_NONE 0
#define O3DML_ACT_RELU 1
#define O3DML_ACT_LEAKY 2

O3DML_API int o3dml_abi_version(void);
O3DML_API const char* o3dml_last_error(void);
/* number of CUDA kernels this library has enqueued in the process (bench.py: gpu_launches) */
O3DML_API unsigned long long o3dml_launch_count(void);
/* a host that replays kernels of this library from a captured CUDA graph reports them here
 * (the counter above only sees direct launches) */
O3DML_API void o3dml_launch_count_add(unsigned long long n);

/* ------------------------------------------------------------------ ops ---- */

/* open3d.ml.torch.ops.voxelize(points, row_splits, voxel_size, points_range_min,
 * points_range_max, max_points_per_voxel, max_voxels)
 *   call sites: ml3d/torch/models/point_pillars.py:354-357, sparseconvnet.py:293-298.
 * points: float32 rows of `point_stride` floats, xyz first (so `points_feats[:, :3]`
 * needs no copy).  Outputs sized for the worst case (num_points voxels):
 *   voxel_coords int32 [num_points,3] (x,y,z), voxel_point_indices int64 [num_points],
 *   voxel_point_row_splits int64 [num_points+1], voxel_batch_splits int64 [batch+1],
 *   voxel_batch_id int32 [num_points] (optional, may be NULL),
 *   d_counts int64 [2] = {num_voxels, num_kept_points}. */
O3DML_API size_t o3dml_voxelize_workspace_bytes(int64_t num_points, int64_t batch);
O3DML_API int o3dml_voxelize(const float* points, int64_t num_points, int point_stride,
                   const int64_t* row_splits, int64_t batch, const float* h_voxel_size,
                   const float* h_range_min, const float* h_range_max,
                   int64_t max_points_per_voxel, int64_t max_voxels, int32_t* voxel_coords,
                   int64_t* voxel_point_indices, int64_t* voxel_point_row_splits,
                   int64_t* voxel_batch_splits, int32_t* voxel_batch_id, int64_t* d_counts,
                   void* workspace, size_t workspace_bytes, void* stream);

/* open3d.ml.torch.ops.ragged_to_dense(values, row_splits, out_col_size, default_value)
 *   call sites: point_pillars.py:364-366, kpconv.py:2030-2032.
 * values: [L, inner] elements of elem_bytes (4 or 8, integer); out [rows, out_col_size, inner];
 * `add` is added to every output element (fuses the "+ 1" of point_pillars.py:366). */
O3DML_API int o3dml_ragged_to_dense(const void* values, int elem_bytes, int64_t inner,
                          const int64_t* row_splits, int64_t rows, int64_t out_col_size,
                          int64_t fill_bits, int64_t add, void* out, void* stream);

/* open3d.core.nns.NearestNeighborSearch(points).knn_search(queries, k)
 *   (ml3d/datasets/utils/dataprocessing.py:99-103 <- randlanet.py:218-229) and
 * open3d.ml.torch.ops.knn_search(points, queries, k, points_row_splits, queries_row_splits,
 *   return_distances) (ml3d/torch/models/point_transformer.py:724-734).
 * out_index [num_queries, k] int32 or int64 GLOBAL row ids (-1 when a batch item has fewer than
 * k points), out_distance2 [num_queries, k] float32 squared distances (may be NULL).
 * Rows ascend by (distance, index). */
O3DML_API size_t o3dml_knn_workspace_bytes(int64_t num_points, int64_t num_queries, int64_t batch);
O3DML_API int o3dml_knn_search(const float* points, int64_t num_points, const int64_t* points_row_splits,
                     const float* queries, int64_t num_queries,
                     const int64_t* queries_row_splits, int64_t batch, int k, void* out_index,
                     int index_is64, float* out_distance2, void* workspace,
                     size_t workspace_bytes, void* stream);

/* open3d.ml.torch.layers.FixedRadiusSearch()(points, queries, radius, points_row_splits,
 *   queries_row_splits)  (ml3d/torch/models/kpconv.py:2021-2026), two phases:
 *   count: neighbors_row_splits int64 [num_queries+1], d_total int64 [1];
 *   fill : neighbors_index int32 [total] (global ids), neighbors_distance2 float32 [total];
 * the workspace must be left untouched between the two calls. */
O3DML_API size_t o3dml_radius_workspace_bytes(int64_t num_points, int64_t num_queries, int64_t batch);
O3DML_API int o3dml_radius_count(const float* points, int64_t num_points, const int64_t* points_row_splits,
                       const float* queries, int64_t num_queries,
                       const int64_t* queries_row_splits, int64_t batch, float radius,
                       int64_t* neighbors_row_splits, int64_t* d_total, void* workspace,
                       size_t workspace_bytes, void* stream);
O3DML_API int o3dml_radius_fill(const float* queries, int64_t num_points, int64_t num_queries,
                      const int64_t* queries_row_splits, int64_t batch, float radius,
                      const int64_t* neighbors_row_splits, int32_t* neighbors_index,
                      float* neighbors_distance2, void* workspace, size_t workspace_bytes,
                      void* stream);

/* Distance metrics of the general searches below (DESIGN.md section 2): with d = query - point per axis,
 * L2 = (dx*dx + dy*dy) + dz*dz (returned squared), L1 = (|dx| + |dy|) + |dz|, LINF = max(max(|dx|, |dy|), |dz|),
 * all in float32 without FMA.  Rows ascend by (distance, index). */
#define O3DML_METRIC_L2 0
#define O3DML_METRIC_L1 1
#define O3DML_METRIC_LINF 2

/* open3d.ml.torch.ops.fixed_radius_search / radius_search and layers.FixedRadiusSearch / RadiusSearch with every
 * option: the two phases of o3dml_radius_count / _fill (same workspace, o3dml_radius_workspace_bytes, left untouched
 * between them), which are their L2 / one-radius / int32 case.  A point is kept when distance <= t, t = r * r for L2
 * and r otherwise.  radii float32 [num_queries] (may be NULL: every query takes `radius`, which must be > 0): a
 * negative, NaN or infinite radius gives an empty row.  ignore_query_point skips every point whose three coordinates
 * equal the query's.  Both phases take the same radius, radii, metric and ignore_query_point.  Fill: neighbors_index
 * int32 or int64 (index_is64) [total]; neighbors_distance float32 [total], divided by t (L2) or r (L1, LINF) under
 * normalize_distances. */
O3DML_API int o3dml_radius_search_count(const float* points, int64_t num_points, const int64_t* points_row_splits,
                                        const float* queries, int64_t num_queries,
                                        const int64_t* queries_row_splits, int64_t batch, float radius,
                                        const float* radii, int metric, int ignore_query_point,
                                        int64_t* neighbors_row_splits, int64_t* d_total, void* workspace,
                                        size_t workspace_bytes, void* stream);
O3DML_API int o3dml_radius_search_fill(const float* queries, int64_t num_points, int64_t num_queries,
                                       const int64_t* queries_row_splits, int64_t batch, float radius,
                                       const float* radii, int metric, int ignore_query_point,
                                       int normalize_distances, const int64_t* neighbors_row_splits,
                                       void* neighbors_index, int index_is64, float* neighbors_distance,
                                       void* workspace, size_t workspace_bytes, void* stream);

/* open3d.ml.torch.ops.knn_search / layers.KNNSearch with a metric and ignore_query_point; o3dml_knn_search is its
 * L2 case without ignore_query_point.  Without ignore_query_point: out_index [num_queries, k] and out_distance
 * [num_queries, k] (may be NULL) as there, out_row_splits and d_total unused.  With it a row may hold fewer than k
 * neighbours: out_index / out_distance hold the rows back to back (room for num_queries * k entries),
 * out_row_splits int64 [num_queries + 1] places them and d_total (int64 [1], may be NULL) is their total. */
O3DML_API size_t o3dml_knn_search_metric_workspace_bytes(int64_t num_points, int64_t num_queries, int64_t batch,
                                                         int k, int ignore_query_point);
O3DML_API int o3dml_knn_search_metric(const float* points, int64_t num_points, const int64_t* points_row_splits,
                                      const float* queries, int64_t num_queries, const int64_t* queries_row_splits,
                                      int64_t batch, int k, int metric, int ignore_query_point, void* out_index,
                                      int index_is64, float* out_distance, int64_t* out_row_splits,
                                      int64_t* d_total, void* workspace, size_t workspace_bytes, void* stream);

/* Per-voxel reduction over the CSR voxel lists of o3dml_voxelize: the second half of
 *   open3d.ml.contrib.subsample / subsample_batch (barycentre grid subsampling,
 *   ml3d/datasets/utils/dataprocessing.py:14-49, ml3d/torch/models/kpconv.py:2037-2164) and of
 *   open3d.ml.torch.ops.voxel_pooling (position_fn / feature_fn in {average, max, nearest}).
 * out_points [M,3] (may be NULL), out_features [M,F], out_labels [M] int32 = most frequent label of the
 * voxel (ties: smallest).  Modes: 0 mean (sequential fp32 sum in ascending point id, then one divide),
 * 1 max, 2 first point of the voxel.  d_num_voxels may be NULL (= num_voxels_bound). */
O3DML_API int o3dml_voxel_reduce(const float* points, int point_stride, const float* features,
                                 int feat_channels, int feat_stride, const int32_t* labels,
                                 const int64_t* voxel_row_splits, const int64_t* voxel_point_indices,
                                 const int64_t* d_num_voxels, int64_t num_voxels_bound, int position_mode,
                                 int feature_mode, float* out_points, float* out_features,
                                 int32_t* out_labels, void* stream);

/* open3d.ml.torch.ops.reduce_subarrays_sum(values, row_splits) (ml3d/torch/models/sparseconvnet.py:318-324):
 * out[i] = sum(values[row_splits[i] : row_splits[i+1]]), float32, sequential adds in index order. */
O3DML_API int o3dml_reduce_subarrays_sum(const float* values, const int64_t* row_splits, int64_t num_rows,
                                         float* out, void* stream);

/* ------------------------------------------------------- PointPillars ---- */

/* PillarFeatureNet.forward + PFNLayer.forward + PointPillarsScatter.forward fused
 *   (point_pillars.py:512-555, 417-453, 577-616), consuming the CSR voxel lists of
 *   o3dml_voxelize directly (no [M,32,C] pillar tensor).  w_t [C+5, 64] = linear.weight^T,
 *   bn_scale/shift = folded eval BatchNorm1d(eps 1e-3).  Pillars with x >= nx or y >= ny are
 *   skipped for the canvas (point_pillars.py:373-380).  feat_out [M,64] and canvas may be NULL;
 *   canvas is NHWC [B,ny,nx,64] or NCHW [B,64,ny,nx] and must be zero-filled by the caller.
 *   d_num_voxels: device count (d_counts of o3dml_voxelize); num_voxels_bound: host upper bound. */
O3DML_API int o3dml_pp_pfn_scatter(const float* points, int point_stride, int point_channels,
                         const int32_t* voxel_coords, const int64_t* voxel_row_splits,
                         const int64_t* voxel_point_indices, const int32_t* voxel_batch_id,
                         const int64_t* d_num_voxels, int64_t num_voxels_bound, const float* w_t,
                         const float* bn_scale, const float* bn_shift, int out_channels, float vx,
                         float vy, float x_offset, float y_offset, int nx, int ny,
                         int max_points_per_voxel, float* feat_out, float* canvas,
                         int canvas_nchw, void* stream);

/* o3dml_pp_pfn_scatter for the two-layer PillarFeatureNet (feat_channels [64, 64], e.g. the nuScenes and Argoverse
 *   configs): layer 0 w0_t [C+5, 32] with folded BN bn0_scale/shift [32], then layer 1 w1_t [64, 64] =
 *   linear.weight^T with folded BN bn1_scale/shift [64] on [y0 | max over slots of y0] (point_pillars.py:400-453).
 *   Every slot takes part in both maxima; only layer 0's input is masked, so a padded slot's layer-1 value is
 *   relu(BN1(W1 . [relu(BN0(0)) | m0])), which differs per pillar.  Other arguments and checks as above. */
O3DML_API int o3dml_pp_pfn2_scatter(const float* points, int point_stride, int point_channels,
                         const int32_t* voxel_coords, const int64_t* voxel_row_splits,
                         const int64_t* voxel_point_indices, const int32_t* voxel_batch_id,
                         const int64_t* d_num_voxels, int64_t num_voxels_bound, const float* w0_t,
                         const float* bn0_scale, const float* bn0_shift, const float* w1_t,
                         const float* bn1_scale, const float* bn1_shift, int out_channels, float vx,
                         float vy, float x_offset, float y_offset, int nx, int ny,
                         int max_points_per_voxel, float* feat_out, float* canvas, int canvas_nchw,
                         void* stream);

/* Neighbour table of open3d.ml.torch.layers.SparseConv / SparseConvTranspose
 *   (ml3d/torch/models/sparseconvnet.py:344-485): neighbors int32 [num_out, kx*ky*kz] = id of the input point
 *   in kernel cell (x, y, z) (row-major, the layout of the layer's `kernel` parameter [kx, ky, kz, Cin, Cout])
 *   of each output, or num_in when the cell is empty; neighbor_count int32 [num_out] (may be NULL) = non-empty
 *   cells (the `normalize` divisor).  cell_a = floor((in_a - out_a) / voxel_size + offset_a + ks_a / 2), with
 *   in / out swapped for the transposed convolution.  The contraction is o3dml_linear(_tc) with the table
 *   columns as index operands. */
O3DML_API size_t o3dml_sparse_conv_workspace_bytes(int64_t num_in);
O3DML_API int o3dml_sparse_conv_neighbors(const float* in_positions, int64_t num_in,
                                          const float* out_positions, int64_t num_out, float voxel_size,
                                          const float* h_offset, const int* h_kernel_size, int transpose,
                                          int32_t* neighbors, int32_t* neighbor_count, void* workspace,
                                          size_t workspace_bytes, void* stream);

/* open3d.ml.torch.ops.continuous_conv (op surface named by the north star; no call site in the reference):
 *   out[o] = sum_n imp_n * W(map((inp_pos[n] - out_pos[o]) * 2 / extent + offset))^T f[n] over the neighbour list
 *   [neighbors_row_splits[o], neighbors_row_splits[o+1]) of neighbors_index; filters [size_z, size_y, size_x, Cin, Cout];
 *   coordinate_mapping 0 identity / 1 ball_to_cube_radial; interpolation 0 nearest / 1 linear (clamped) /
 *   2 linear_border (zero outside); normalize divides by the sum of the importances (or the neighbour count). */
O3DML_API int o3dml_continuous_conv(const float* filters, int size_x, int size_y, int size_z, int in_channels,
                                    int out_channels, const float* out_positions, int64_t num_out,
                                    const float* extents, int extents_per_point, const float* h_offset,
                                    const float* inp_positions, const float* inp_features, int64_t num_inp,
                                    const float* inp_importance, const void* neighbors_index, int index_is64,
                                    const float* neighbors_importance, const int64_t* neighbors_row_splits,
                                    int align_corners, int coordinate_mapping, int normalize, int interpolation,
                                    float* out, void* stream);

/* open3d.ml.torch.ops.continuous_conv_transpose (op surface named by the north star; no call site in the reference),
 *   the exact adjoint of o3dml_continuous_conv: for output j with the inputs i = neighbors_index[e] of its list
 *   [neighbors_row_splits[j], neighbors_row_splits[j+1]),
 *   out[j] = oimp_j * sum_e nimp_e * s_i * W(map((out_pos[j] - inp_pos[i]) * 2 / extent_i + offset))^T f[i]
 *   with extent_i = extents[extents_per_point ? i : 0], oimp = out_importance and nimp = neighbors_importance (NULL:
 *   ones), s_i = 1 / inp_neighbors_importance_sum[i] under normalize (NULL: 1 / the length of row i of
 *   inp_neighbors_row_splits; one of the two is required), 1 for a zero divisor and without normalize.  Filter
 *   layout, mapping, interpolation and limits as in o3dml_continuous_conv; fp32 sums in list order.  inp_positions /
 *   inp_features may be NULL when num_inp == 0. */
O3DML_API int o3dml_continuous_conv_transpose(const float* filters, int size_x, int size_y, int size_z,
                                              int in_channels, int out_channels, const float* out_positions,
                                              int64_t num_out, const float* out_importance, const float* extents,
                                              int extents_per_point, const float* h_offset,
                                              const float* inp_positions, const float* inp_features, int64_t num_inp,
                                              const float* inp_neighbors_importance_sum,
                                              const int64_t* inp_neighbors_row_splits, const void* neighbors_index,
                                              int index_is64, const float* neighbors_importance,
                                              const int64_t* neighbors_row_splits, int align_corners,
                                              int coordinate_mapping, int normalize, int interpolation, float* out,
                                              void* stream);

/* open3d.ml.torch.ops.invert_neighbors_list(num_points, inp_neighbors_index, inp_neighbors_row_splits,
 *   inp_neighbors_attributes) (no call site in the reference; pairs with the transposed convolution above):
 *   num_inp rows of num_entries ids in [0, num_points) regrouped by id.  neighbors_index [num_entries] (int32 or
 *   int64, as the input) holds, for every row j, the input rows i that contain j, once per occurrence, ordered by
 *   (i, position in row i): a stable sort of the entries by id.  neighbors_row_splits int64 [num_points + 1].
 *   Entries whose id is out of range are dropped: they follow the last row, in input order, and
 *   neighbors_row_splits[num_points] counts the entries kept.  permutation int64 [num_entries]: the input entry at
 *   each output position (the caller permutes per-entry attributes with it).  num_entries < 2^32. */
O3DML_API size_t o3dml_invert_neighbors_list_workspace_bytes(int64_t num_entries);
O3DML_API int o3dml_invert_neighbors_list(int64_t num_points, const void* inp_neighbors_index, int index_is64,
                                          const int64_t* inp_neighbors_row_splits, int64_t num_inp,
                                          int64_t num_entries, void* neighbors_index, int64_t* neighbors_row_splits,
                                          int64_t* permutation, void* workspace, size_t workspace_bytes,
                                          void* stream);

/* ------------------------------------------- detection post-processing ---- */

/* open3d.ml.torch.ops.nms(boxes, scores, nms_overlap_thresh) -- rotated-BEV greedy NMS
 *   (ml3d/torch/utils/objdet_helper.py:346 <- multiclass_nms <- Anchor3DHead.get_bboxes_single,
 *   ml3d/torch/models/point_pillars.py:967-1025).  boxes [N,5] = (x0, y0, x1, y1, r): the rectangle
 *   [x0,x1]x[y0,y1] rotated by r about its centre.  keep_indices int64 [N] receives the kept original
 *   indices by descending score (ties: lower index first), d_num_keep int64 [1] their count. */
O3DML_API size_t o3dml_nms_workspace_bytes(int64_t num_boxes);
O3DML_API int o3dml_nms(const float* boxes, const float* scores, int64_t num_boxes, float iou_threshold,
                        int64_t* keep_indices, int64_t* d_num_keep, void* workspace,
                        size_t workspace_bytes, void* stream);

/* open3d.ml.contrib.iou_bev_{cpu,cuda} (mode 0: boxes [.,5] = (x, y, w, h, r)) and iou_3d_{cpu,cuda}
 *   (mode 1: boxes [.,7] = (x, y, z, w, h, l, ry), ground plane (x, z), vertical span [y - h, y]):
 *   out [num_a, num_b] float32 IoU (ml3d/metrics/mAP.py:85-89, ml3d/datasets/utils/operations.py:430). */
O3DML_API int o3dml_iou_matrix(const float* boxes_a, int64_t num_a, const float* boxes_b, int64_t num_b,
                               int mode, float* out, void* stream);

/* PointPillars box decoding (Anchor3DHead.get_bboxes, ml3d/torch/models/point_pillars.py:945-1025) for a batch of
 *   frames, contract in DESIGN.md section 2.  cls [B, A*C, H, W], reg [B, A*7, H, W], dir [B, A*2, H, W]: NCHW with
 *   contiguous H x W planes, frame b at map + b * <map>_batch_stride floats.  anchors [H*W*A, 7] float32 are the
 *   reference's grid_anchors for this (H, W) (row (y * W + x) * A + a).  With K = min(nms_pre, H*W*A) the outputs
 *   are boxes [B, C*K, 7], scores [B, C*K], labels int64 [B, C*K] (rows at or past d_counts[b] are zero, label -1)
 *   and d_counts int64 [B].  nms_pre is at most 4096.  No host synchronisation; capturable into a CUDA graph. */
O3DML_API size_t o3dml_pp_detect_workspace_bytes(int64_t batch, int64_t height, int64_t width, int num_anchors,
                                                 int num_classes, int64_t nms_pre);
O3DML_API int o3dml_pp_detect(const float* cls, int64_t cls_batch_stride, const float* reg, int64_t reg_batch_stride,
                              const float* dir, int64_t dir_batch_stride, int64_t batch, int64_t height,
                              int64_t width, int num_anchors, int num_classes, const float* anchors, int64_t nms_pre,
                              float score_thr, float dir_offset, float* out_boxes, float* out_scores,
                              int64_t* out_labels, int64_t* d_counts, void* workspace, size_t workspace_bytes,
                              void* stream);

/* ------------------------------------------------------ dense layers ---- */

/* One operand of the gathered GEMM: rows of `channels` floats (row stride ld); when `index`
 * is given, output row n reads row index[n * index_ld], index_ld <= 0 reading as 1 (ids outside [0, rows) read zeros:
 * the "shadow" neighbours of kpconv.py:821-858); with out_rows_per_batch > 0 the ids are
 * relative to the batch item n / out_rows_per_batch (RandLA-Net's [B,N,1] interp_idx). */
typedef struct o3dml_src_t {
    const float* data;
    const void* index;
    int64_t rows;
    int64_t out_rows_per_batch;
    int64_t src_rows_per_batch;
    int32_t channels;
    int32_t ld;
    int32_t index_is64;
    int32_t index_ld;
} o3dml_src_t;

/* out[n, :] = act(scale * (concat_s src_s[n] @ weight_t) + shift + residual[n, :])
 *   SharedMLP (randlanet.py:471-518), decoder concat + nearest_interpolation
 *   (randlanet.py:284-292, 329-350), UnaryBlock / closest_pool (kpconv.py:1255-1295, 821-837),
 *   Anchor3DHead 1x1 convs (point_pillars.py:827-841).
 * weight_t [sum channels, out_channels] row-major; scale/shift/residual may be NULL.
 * out_nchw_plane > 0 writes out[(n / plane), c, (n % plane)] instead of row-major. */
O3DML_API int o3dml_linear(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs, const float* weight_t,
                 const float* scale, const float* shift, const float* residual, int residual_ld,
                 int act, float slope, float* out, int out_ld, int out_channels,
                 int out_nchw_plane, void* stream);

/* 3x3 convolution, padding 1, stride 1|2, NHWC, + folded BN + activation
 *   (SECOND blocks, point_pillars.py:641-667).  weight_t [(ky*3+kx)*C + c, out_channels]. */
O3DML_API int o3dml_conv3x3_nhwc(const float* in, int batch, int H, int W, int C, int stride,
                       const float* weight_t, const float* scale, const float* shift, int act,
                       float slope, float* out, int out_channels, void* stream);

/* ConvTranspose2d with kernel == stride (SECONDFPN deblocks, point_pillars.py:707-755), NHWC;
 * writes out_channels channels at out (row stride out_ld: the 384-channel concat buffer).
 * weight_t [C, (ky*s+kx)*out_channels + co]; scale/shift tiled to [s*s*out_channels]. */
O3DML_API int o3dml_deconv_nhwc(const float* in, int batch, int H, int W, int C, int stride,
                      const float* weight_t, const float* scale, const float* shift, int act,
                      float slope, float* out, int out_ld, int out_channels, void* stream);

/* Tensor-core (wgmma TF32, 3xTF32 split: ~2^-21 relative per product) variants of the three
 * dense entry points above.  Instead of weight_t they take the host-packed TF32 hi/lo image of the
 * weight: fp32 [2 * n_pad][k_pad] row-major, rows [0, n_pad) = tf32(w[:, n]) and rows [n_pad, 2 n_pad) =
 * tf32(w - hi) (zero padded; k_pad % 32 == 0; n_pad in {32, 64, 128*j}; 16-byte aligned;
 * open3d_ml_b200._lib.pack_linear).  Identity sources and convolution taps are fetched with
 * cp.async.bulk.tensor (the library encodes the tensor maps per call), gathered sources with cp.async.
 * Contract on the sources (o3dml_linear_tc_supported returns 1 when it holds): channels % 4 == 0,
 * ld % 4 == 0, 16-byte aligned data, and channels % 32 == 0 for every source but the last;
 * o3dml_conv3x3_nhwc_tc needs C % 32 == 0. */
O3DML_API int o3dml_linear_tc_supported(const o3dml_src_t* srcs, int num_srcs);
O3DML_API int o3dml_linear_tc(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs,
                              const void* weight_image, int k_pad, int n_pad, const float* scale,
                              const float* shift, const float* residual, int residual_ld, int act,
                              float slope, float* out, int out_ld, int out_channels,
                              int out_nchw_plane, void* stream);
O3DML_API int o3dml_conv3x3_nhwc_tc(const float* in, int batch, int H, int W, int C, int stride,
                                    const void* weight_image, int k_pad, int n_pad, const float* scale,
                                    const float* shift, int act, float slope, float* out,
                                    int out_channels, void* stream);
O3DML_API int o3dml_deconv_nhwc_tc(const float* in, int batch, int H, int W, int C, int stride,
                                   const void* weight_image, int k_pad, int n_pad, const float* scale,
                                   const float* shift, int act, float slope, float* out, int out_ld,
                                   int out_channels, void* stream);

/* Narrow per-point dense layer, one thread per row (rowmlp.cu): same contract as o3dml_linear
 * for 1 or 2 sources (the second may be gathered) without residual / NCHW output, for the
 * (channels0, channels1, out_channels) triples listed in csrc/rowmlp_shapes.inc
 * (o3dml_linear_rows_small_supported returns 1 for those).  weight_t [K, out_channels], scale and
 * shift (may be NULL) are read from HOST memory at call time and travel in the kernel parameter
 * block, so every multiply takes its weight from the constant bank: these layers
 * (SharedMLPs of RandLA-Net's first level and classifier, randlanet.py:110-113, :653-664) are
 * HBM-bound and need neither shared memory nor barriers. */
O3DML_API int o3dml_linear_rows_small_supported(int channels0, int channels1, int out_channels);
O3DML_API int o3dml_linear_rows_small(int64_t num_rows, const o3dml_src_t* srcs, int num_srcs,
                                      const float* h_weight_t, const float* h_scale,
                                      const float* h_shift, int act, float slope, float* out, int out_ld,
                                      int out_channels, void* stream);

/* ---------------------------------------------------------- RandLA-Net ---- */

/* LocalSpatialEncoding + AttentivePooling score/softmax/sum fused (randlanet.py:521-639, as
 * used by LocalFeatureAggregation.forward :667-692).  stage 1: X = [feat[nbr] | r1];
 * stage 2: X = [feat[nbr] | lrelu(BN(wl2 r1))].  feat [B*N, d/2]; agg out [B*N, d].
 * w10_t [10, d/2], wl2_t [d/2, d/2], wscore_t [d, d] are [in, out]; s, t = folded BN(+bias).
 * d in {16, 32, 64, 128, 256, 512}, all on the tiled FP32 SIMT kernel. */
O3DML_API int o3dml_randla_lfa_pool(int stage, int d, const float* coords, const void* neighbor_idx,
                          int idx_is64, int num_neighbors, const float* feat, int64_t batch,
                          int64_t n_per_batch, const float* w10_t, const float* s10,
                          const float* t10, const float* wl2_t, const float* s2, const float* t2,
                          const float* wscore_t, const float* bscore, float* agg, void* stream);

/* d = 16 variant of o3dml_randla_lfa_pool (the first, largest RandLA-Net level) that takes the
 * layer's weights from HOST memory, packed as O3DML_LFA16_WEIGHT_FLOATS floats:
 *   [0,80) w10_t [10][8] | [80,88) s10 | [88,96) t10 | [96,160) wl2_t [8][8] | [160,168) s2 |
 *   [168,176) t2 | [176,432) wscore_t [16][16] | [432,448) bscore        (all [in][out])
 * They travel in the kernel parameter block, so every FMA reads its weight as a constant-bank
 * operand (no shared-memory broadcast loads).  Stage 1 ignores the wl2/s2/t2 fields. */
#define O3DML_LFA16_WEIGHT_FLOATS 448
O3DML_API int o3dml_randla_lfa16_pool(int stage, const float* coords, const void* neighbor_idx, int idx_is64,
                                      int num_neighbors, const float* feat, int64_t batch,
                                      int64_t n_per_batch, const float* h_weights, float* agg,
                                      void* stream);

/* Tensor-core (wgmma fp16, 3xFP16 split) variant of o3dml_randla_lfa_pool, same contract, d in
 * {16, 32, 64, 128, 256}.  wscore_image / wl2_image: the weight [out][in] packed by the host as
 * fp16 hi/lo operand images in the chunk-major layout ([in/8][out][8 halves] hi, then the
 * same for lo; open3d_ml_b200._lib.pack_operand_image); wl2_t (fp32 [in][out]) is used instead of
 * wl2_image when d == 16.  The score bias cancels in the softmax and is not taken. */
O3DML_API int o3dml_randla_lfa_pool_tc(int stage, int d, const float* coords, const void* neighbor_idx,
                                       int idx_is64, int num_neighbors, const float* feat, int64_t batch,
                                       int64_t n_per_batch, const float* w10_t, const float* s10,
                                       const float* t10, const void* wl2_image, const float* wl2_t,
                                       const float* s2, const float* t2, const void* wscore_image,
                                       float* agg, void* stream);

/* The per-point tail of RandLA-Net in one kernel: last decoder SharedMLP on [skip | nearest_interpolation(x)]
 * (randlanet.py:284-292, 329-350) + the fc1 classifier stack (randlanet.py:110-113, 294-298), four dense layers
 * 32+32 -> 32 -> 64 -> 32 -> classes chained through shared memory (wgmma TF32, 3xTF32).
 * weight_image: 57 344-byte device image of the four weights (open3d_ml_b200._lib.pack_tail_image: per layer and
 * 32-wide k-chunk, TF32 hi tiles then lo tiles of [N][32] floats, K-major SWIZZLE_128B); h_scale / h_shift: HOST float
 * [4][64] folded BN scale / shift (+ bias) per layer; LeakyReLU(slope) after the first three layers.
 * interp_index [num_rows] (int32 / int64).  Row n reads coarse row r = interp_index[n] when out_rows_per_batch == 0
 * (global), r = interp_index[n] + (n / out_rows_per_batch) * src_rows_per_batch when out_rows_per_batch > 0
 * (batch-relative).  The coarse half of row n is zero when interp_index[n] < 0, when interp_index[n] >=
 * src_rows_per_batch (batch-relative), or when r >= coarse_rows.  skip_ld / coarse_ld: row strides in floats, multiples
 * of 4 with 16-byte aligned rows.  classes 1..32.  out [num_rows, classes], exactly num_rows rows written; num_rows
 * <= 0 returns without a launch. */
O3DML_API int o3dml_randla_tail_supported(int skip_channels, int coarse_channels, int c1, int c2, int c3, int classes);
O3DML_API int o3dml_randla_tail(const float* skip, int skip_ld, const float* coarse, int coarse_ld,
                                int64_t coarse_rows, const void* interp_index, int index_is64,
                                int64_t out_rows_per_batch, int64_t src_rows_per_batch, int64_t num_rows,
                                const void* weight_image, const float* h_scale, const float* h_shift, float slope,
                                int classes, float* out, void* stream);

/* out[n, :] = max_j src[index[n, j], :]  -- RandLANet.random_sample (randlanet.py:300-327),
 * KPConv max_pool (kpconv.py:840-858, shadow_zero = 1), k = 1: nearest_interpolation /
 * closest_pool. */
O3DML_API int o3dml_gather_max(const float* src, int64_t src_rows, int channels, int src_ld,
                     const void* index, int index_is64, int64_t num_rows, int k,
                     int64_t out_rows_per_batch, int64_t src_rows_per_batch, int shadow_zero,
                     float* out, int out_ld, void* stream);

/* -------------------------------------------------------------- KPConv ---- */

/* Neighbour gather + kernel-point (linear) influence of KPConv.forward (kpconv.py:1044-1147):
 * weighted_features [num_queries, K*Cin] with [n, k*Cin + c] = sum_h max(0, 1 - |nb_h - q - kp_k|
 * / extent) * features[idx[n,h], c]; the [K*Cin, Cout] contraction is o3dml_linear. */
O3DML_API int o3dml_kpconv_gather(const float* query_points, int64_t num_queries,
                        const float* support_points, int64_t num_support,
                        const void* neighbor_index, int index_is64, int max_neighbors,
                        const float* features, int in_channels, const float* kernel_points,
                        int num_kernel_points, float kp_extent, float* weighted_features,
                        void* stream);

/* The same operand for a deformable KPConv (kpconv.py:1011-1106, modulated = False): query n uses the
 * kernel points kp_k + kp_extent * offsets[n * offset_ld + 3k .. 3k+2] (product, then sum, each rounded
 * in fp32).  A neighbour is kept when |nb_h - q - kp_k|^2 < kp_extent^2 for some k; dropped neighbours
 * contribute nothing (their features are never read, so a non-finite one does not propagate), kept
 * neighbours contribute for every k and are summed in ascending h.  offsets is [num_queries, offset_ld]
 * with offset_ld >= 3K.  Supports in_channels % 4 == 0 with 16-byte aligned features / output, or
 * in_channels <= 8; anything else is rejected. */
O3DML_API int o3dml_kpconv_gather_deformable(const float* query_points, int64_t num_queries,
                        const float* support_points, int64_t num_support,
                        const void* neighbor_index, int index_is64, int max_neighbors,
                        const float* features, int in_channels, const float* kernel_points,
                        int num_kernel_points, float kp_extent, const float* offsets, int offset_ld,
                        float* weighted_features, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3DML_B200_H */
