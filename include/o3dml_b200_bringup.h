/*
 * o3dml_b200_bringup.h -- wgmma bring-up / profiling hooks of libo3dml_b200.so.  NOT part of the product ABI
 * (include/o3dml_b200.h): used by tests/test_gpu_tc.py to pin the descriptor encodings and the 3xFP16 operand layout of
 * csrc/tc.cuh.
 */
#ifndef O3DML_B200_BRINGUP_H
#define O3DML_B200_BRINGUP_H
#include "o3dml_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* wgmma regression hook: d[128, n] = a[128, k] * b[n, k]^T on the tensor cores with the
 * 3xFP16 split used by the fused kernels (terms = 1: hi*hi only).  One CTA (one warpgroup); n, k multiples of 16. */
O3DML_API int o3dml_tc_gemm_test(const float* a, const float* b, float* d, int n, int k, int terms,
                                 void* stream);

/* wgmma issue-rate probe (profiling aid): reps x N/16 x 6 MMAs of M=64 x 16 x K=16; out[0] = total cycles,
 * out[1] = cycles spent issuing. */
O3DML_API int o3dml_tc_mma_rate(int n, int reps, long long* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* O3DML_B200_BRINGUP_H */
