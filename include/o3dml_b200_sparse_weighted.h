/* o3dml_b200_sparse_weighted.h -- the weighted sparse-convolution contraction of the C ABI of libo3dml_b200.so, behind
 * open3d.ml.torch.ops.sparse_conv / sparse_conv_transpose with importances and the `inp_importance` /
 * `out_importance` arguments of layers.SparseConv / SparseConvTranspose.  Conventions (status return,
 * o3dml_last_error, device pointers, the stream argument, O3DML_ABI_VERSION) are those of o3dml_b200.h, which this
 * header includes.  The entry takes no workspace.  open3d_ml_b200._lib.SPARSE_WEIGHTED_EXPORTS binds exactly what is
 * declared here (tests/test_abi_sparse_weighted.py). */
#ifndef O3DML_B200_SPARSE_WEIGHTED_H
#define O3DML_B200_SPARSE_WEIGHTED_H
#include "o3dml_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* o3dml_sparse_conv_tc (o3dml_b200_sparseconvunet.h) with a weight per table entry, in one tensor-core launch:
 *   out[m, :] = act(scale * sum_c W_c^T (w[m, c] * pre(features[table[m, c], :])) + shift + residual[m, :]),
 * m < num_out, c < cells, with entry_weight w float [num_out, weight_ld], weight_ld >= cells, parallel to the table.
 * The weight multiplies after the prologue pre(x) and before the 3xTF32 split, so a power-of-two weight scales the
 * product exactly (away from the subnormal range) and a weight of one gives o3dml_sparse_conv_tc's result bit for
 * bit.  A shadow entry contributes zero whatever its weight (also Inf or NaN).  Every other argument, limit and
 * refusal is that of o3dml_sparse_conv_tc; num_out == 0 returns without a launch. */
O3DML_API int o3dml_sparse_conv_weighted_tc(int64_t num_out, const float* features, int64_t num_in, int channels,
                                            int features_ld, const int32_t* table, int cells, int table_ld,
                                            const float* pre_scale, const float* pre_shift, const void* weight_image,
                                            int k_pad, int n_pad, const float* scale, const float* shift,
                                            const float* residual, int residual_ld, int act, float slope, float* out,
                                            int out_ld, int out_channels, const float* entry_weight, int weight_ld,
                                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3DML_B200_SPARSE_WEIGHTED_H */
