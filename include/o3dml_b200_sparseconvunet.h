/* o3dml_b200_sparseconvunet.h -- the sparse-convolution contraction of the C ABI of libo3dml_b200.so, behind
 * open3d.ml.torch.layers.SparseConv / SparseConvTranspose, ops.sparse_conv and the fused SparseConvUnet forward.
 * Conventions (status return, o3dml_last_error, device pointers, the stream argument, O3DML_ABI_VERSION) are those of
 * o3dml_b200.h, which this header includes.  The entry takes no workspace.  open3d_ml_b200._lib.SPARSECONVUNET_EXPORTS
 * binds exactly what is declared here (tests/test_abi_sparseconvunet.py). */
#ifndef O3DML_B200_SPARSECONVUNET_H
#define O3DML_B200_SPARSECONVUNET_H
#include "o3dml_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One tensor-core launch (3xTF32, as o3dml_linear_tc) of
 *   out[m, :] = act(scale * sum_c W_c^T pre(features[table[m, c], :]) + shift + residual[m, :]),   m < num_out,
 * over the cells c < cells of an int32 neighbour table [num_out, table_ld] such as o3dml_sparse_conv_neighbors
 * writes.  An id outside [0, num_in) is a shadow id: its row is zero and stays zero through the prologue.
 * pre(x) = relu(pre_scale * x + pre_shift) per input channel when pre_scale / pre_shift are given (both or neither),
 * x otherwise.  features [num_in, features_ld]: channels used, features_ld a multiple of 4 and rows 16-byte aligned.
 * weight_image: the TF32 hi / lo image (as o3dml_linear_tc takes it) of the [cells * Cp, out_channels] matrix whose
 * row c * Cp + i is W_c[i], Cp = channels rounded up to 32 (rows past channels zero); k_pad = cells * Cp.  cells <=
 * 512.  scale / shift / residual may be NULL; act 0 none, 1 relu, 2 leaky relu (slope).  num_out == 0 returns without
 * a launch. */
O3DML_API int o3dml_sparse_conv_tc(int64_t num_out, const float* features, int64_t num_in, int channels,
                                   int features_ld, const int32_t* table, int cells, int table_ld,
                                   const float* pre_scale, const float* pre_shift, const void* weight_image,
                                   int k_pad, int n_pad, const float* scale, const float* shift,
                                   const float* residual, int residual_ld, int act, float slope, float* out,
                                   int out_ld, int out_channels, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3DML_B200_SPARSECONVUNET_H */
