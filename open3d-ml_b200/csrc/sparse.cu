// sparse.cu -- neighbour tables of the voxel-lattice convolutions behind
//   open3d.ml.torch.layers.SparseConv / SparseConvTranspose
//       call sites: ml3d/torch/models/sparseconvnet.py:344-485 (SubmanifoldSparseConv, Convolution, DeConvolution)
// Contract (upstream Open3D is absent: parity unpinned; oracle/ops_ref.c oracle_sparse_conv restates it):
//   SparseConv          cell_a = floor((in_a  - out_a) / voxel_size + offset_a + ks_a / 2)
//   SparseConvTranspose cell_a = floor((out_a - in_a ) / voxel_size + offset_a + ks_a / 2)      a = x, y, z
//   an input contributes kernel[cell_x, cell_y, cell_z]^T f_in to the output when every cell_a lies in [0, ks_a).
// Inputs are voxel-unique lattice points (what InputLayer / calculate_grid produce): the table holds ONE input id
// per (output, kernel cell) -- the lowest id if several inputs share a cell -- or the shadow id N; the contraction
// itself is the gathered GEMM of gemm_tc.cu with the table columns as index operands (no im2col tensor in HBM).
// Integer / latency-bound: inputs are radix-sorted by voxel key once, every (output, cell) is one binary search.
#include "../../include/o3dml_b200.h"
#include "prims.cuh"

namespace o3dml {

__device__ __forceinline__ uint64_t voxel_key(int x, int y, int z) {   // 21 bits per axis, offset keeps negatives ordered
    return ((uint64_t)(uint32_t)(z + (1 << 20)) << 42) | ((uint64_t)(uint32_t)(y + (1 << 20)) << 21) |
           (uint64_t)(uint32_t)(x + (1 << 20));
}

__global__ void sparse_keys_kernel(const float* __restrict__ pos, int64_t n, float inv_v, uint64_t* __restrict__ keys) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = voxel_key((int)floorf(pos[3 * i] * inv_v), (int)floorf(pos[3 * i + 1] * inv_v),
                        (int)floorf(pos[3 * i + 2] * inv_v));
}

struct SparseGeom {
    float inv_v, v;
    float off[3];
    int ks[3];
    int transpose;
};

__device__ __forceinline__ bool sparse_cell_of(const SparseGeom& g, const float* in, const float* out, int* cell) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float d = g.transpose ? (out[a] - in[a]) : (in[a] - out[a]);
        const float r = d * g.inv_v + g.off[a] + 0.5f * (float)g.ks[a];
        const int c = (int)floorf(r);
        if (c < 0 || c >= g.ks[a]) return false;
        cell[a] = c;
    }
    return true;
}

// one thread per (output, kernel cell): the voxel that holds the cell centre, then the exact predicate
__global__ void sparse_neighbors_kernel(const float* __restrict__ in_pos, int64_t n, const float* __restrict__ out_pos,
                                        int64_t m, const uint64_t* __restrict__ skeys, const uint32_t* __restrict__ perm,
                                        SparseGeom g, int32_t* __restrict__ nbr, int32_t* __restrict__ count) {
    const int kc = g.ks[0] * g.ks[1] * g.ks[2];
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m * kc) return;
    const int64_t o = t / kc;
    const int c = (int)(t - o * kc);
    const int cz = c % g.ks[2], cy = (c / g.ks[2]) % g.ks[1], cx = c / (g.ks[2] * g.ks[1]);   // kernel[x][y][z] row-major
    const int cc[3] = {cx, cy, cz};
    const float* op = out_pos + 3 * o;
    int vox[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float rel = ((float)cc[a] + 0.5f - g.off[a] - 0.5f * (float)g.ks[a]) * g.v;   // cell centre
        const float tpos = g.transpose ? op[a] - rel : op[a] + rel;
        vox[a] = (int)floorf(tpos * g.inv_v);
    }
    const uint64_t key = voxel_key(vox[0], vox[1], vox[2]);
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (skeys[mid] < key) lo = mid + 1; else hi = mid;
    }
    int32_t found = (int32_t)n;
    for (int64_t j = lo; j < n && skeys[j] == key; ++j) {     // stable sort: ascending original id inside a voxel
        const uint32_t id = perm[j];
        int cell[3];
        if (sparse_cell_of(g, in_pos + 3 * (size_t)id, op, cell) && cell[0] == cx && cell[1] == cy && cell[2] == cz) {
            found = (int32_t)id;
            break;
        }
    }
    nbr[t] = found;
    if (found != (int32_t)n && count) atomicAdd(&count[o], 1);
}

static RadixSortBufs sparse_carve(Workspace& ws, int64_t num_in) {
    return radix_sort_carve(ws, num_in > 0 ? num_in : 1);
}

}  // namespace o3dml

using namespace o3dml;

extern "C" size_t o3dml_sparse_conv_workspace_bytes(int64_t num_in) {
    return Workspace::measure(sparse_carve, num_in);
}

extern "C" int o3dml_sparse_conv_neighbors(const float* in_positions, int64_t num_in, const float* out_positions,
                                           int64_t num_out, float voxel_size, const float* h_offset,
                                           const int* h_kernel_size, int transpose, int32_t* neighbors,
                                           int32_t* neighbor_count, void* workspace, size_t workspace_bytes,
                                           void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(voxel_size > 0.f && h_offset && h_kernel_size, "sparse_conv: bad geometry");
    O3DML_CHECK(num_in >= 0 && num_out >= 0 && num_in < ((int64_t)1 << 31), "sparse_conv: bad sizes");
    SparseGeom g;
    g.v = voxel_size;
    g.inv_v = 1.0f / voxel_size;
    int kc = 1;
    for (int a = 0; a < 3; ++a) {
        g.off[a] = h_offset[a];
        g.ks[a] = h_kernel_size[a];
        O3DML_CHECK(g.ks[a] >= 1 && g.ks[a] <= 9, "sparse_conv: kernel_size must be in 1..9");
        kc *= g.ks[a];
    }
    g.transpose = transpose ? 1 : 0;
    if (num_out == 0) return O3DML_OK;
    Workspace ws(workspace, workspace_bytes);
    RadixSortBufs b = sparse_carve(ws, num_in);
    O3DML_CHECK_WORKSPACE(ws, "sparse_conv");
    O3DML_CHECK(neighbors && out_positions, "sparse_conv: null output");
    if (neighbor_count) O3DML_CUDA(cudaMemsetAsync(neighbor_count, 0, sizeof(int32_t) * num_out, st));
    if (num_in > 0) {
        O3DML_CUDA(launch<sparse_keys_kernel>((unsigned)ceil_div<int64_t>(num_in, 256), 256, 0, st, in_positions, num_in,
                                              g.inv_v, b.keys_a));
        O3DML_CUDA(radix_sort_pairs(b, true, num_in, 63, st));
    }
    O3DML_CUDA(launch<sparse_neighbors_kernel>((unsigned)ceil_div<int64_t>(num_out * kc, 256), 256, 0, st, in_positions,
                                               num_in, out_positions, num_out, b.keys_a, b.vals_a, g, neighbors,
                                               neighbor_count));
    return O3DML_OK;
}
