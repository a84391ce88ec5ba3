// prims.cuh -- internal device-wide primitives (scan, radix sort).
#pragma once
#include "common.cuh"

namespace o3dml {

// temp of exclusive_scan_u32 over up to n elements
void* scan_carve(Workspace& ws, int64_t n);
cudaError_t exclusive_scan_u32(const uint32_t* in, uint32_t* out, int64_t n, uint32_t* total_out,
                               void* temp, cudaStream_t st);

// scratch of radix_sort_pairs over up to n keys: ping-pong key / value buffers, digit histogram, its scan temp
struct RadixSortBufs {
    uint64_t *keys_a, *keys_b;
    uint32_t *vals_a, *vals_b, *hist;
    void* scan_tmp;
};
RadixSortBufs radix_sort_carve(Workspace& ws, int64_t n);
cudaError_t radix_sort_pairs(RadixSortBufs& b, bool vals_are_iota, int64_t n, int num_bits, cudaStream_t st);

}  // namespace o3dml
