// sparse.cu -- neighbour tables of the voxel-lattice convolutions behind
//   open3d.ml.torch.layers.SparseConv / SparseConvTranspose
//       call sites: ml3d/torch/models/sparseconvnet.py:344-485 (SubmanifoldSparseConv, Convolution, DeConvolution)
// Contract (upstream Open3D is absent: parity unpinned; oracle/ops_ref.c oracle_sparse_conv restates it):
//   SparseConv          cell_a = floor((in_a  - out_a) / voxel_size + offset_a + ks_a / 2)
//   SparseConvTranspose cell_a = floor((out_a - in_a ) / voxel_size + offset_a + ks_a / 2)      a = x, y, z
//   an input contributes kernel[cell_x, cell_y, cell_z]^T f_in to the output when every cell_a lies in [0, ks_a).
// The table holds ONE input id per (output, kernel cell) -- the lowest id if several inputs share a cell -- or the
// shadow id N; the contraction itself is the gathered GEMM of gemm_tc.cu with the table columns as index operands
// (no im2col tensor in HBM).
// Integer / latency-bound: inputs are radix-sorted by voxel key once; every (output, cell) binary-searches the voxels
// its cell box can reach (one on the model's lattices, at most 3 per axis anywhere) and the exact predicate decides.
#include "../../include/o3dml_b200.h"
#include "prims.cuh"

namespace o3dml {

__device__ __forceinline__ uint64_t voxel_key(int x, int y, int z) {   // 21 bits per axis, offset keeps negatives ordered
    return ((uint64_t)(uint32_t)(z + (1 << 20)) << 42) | ((uint64_t)(uint32_t)(y + (1 << 20)) << 21) |
           (uint64_t)(uint32_t)(x + (1 << 20));
}

// the voxel of a coordinate: one rounded product, so the key is a non-decreasing function of the coordinate
__device__ __forceinline__ int voxel_of(float x, float inv_v) { return (int)floorf(__fmul_rn(x, inv_v)); }

__global__ void sparse_keys_kernel(const float* __restrict__ pos, int64_t n, float inv_v, uint64_t* __restrict__ keys) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keys[i] = voxel_key(voxel_of(pos[3 * i], inv_v), voxel_of(pos[3 * i + 1], inv_v), voxel_of(pos[3 * i + 2], inv_v));
}

struct SparseGeom {
    float inv_v, v;
    float off[3];
    int ks[3];
    int transpose;
};

// the kernel cell of an input coordinate on axis a, in the oracle's order: product rounded, + offset, + ks / 2 (no
// fused multiply-add, which would move points that lie on a cell face).  Monotone in the input coordinate:
// non-decreasing, or non-increasing under transpose.
__device__ __forceinline__ int sparse_cell_axis(const SparseGeom& g, int a, float in, float out) {
    const float d = g.transpose ? __fsub_rn(out, in) : __fsub_rn(in, out);
    const float r = __fadd_rn(__fadd_rn(__fmul_rn(d, g.inv_v), g.off[a]), 0.5f * (float)g.ks[a]);
    return (int)floorf(r);
}

// The smallest float whose voxel is >= j: j * v corrected by a few ulp steps.  *exact is cleared when the steps
// run out (the caller then probes the voxel anyway).
__device__ __forceinline__ float voxel_start(int j, float v, float inv_v, bool* exact) {
    float x = __fmul_rn((float)j, v);
    int s = 0;
    for (; s < 8 && voxel_of(x, inv_v) < j; ++s) x = nextafterf(x, INFINITY);
    for (; s < 8 && voxel_of(nextafterf(x, -INFINITY), inv_v) >= j; ++s) x = nextafterf(x, -INFINITY);
    if (s == 8) *exact = false;
    return x;
}

// Bit i of the result: voxel kb - 1 + i on axis a may hold an input whose cell is `cell`.  The cell's box spans one
// voxel width around the voxel kb of its centre, so it reaches kb - 1 .. kb + 1 at most.  Both the voxel and the cell
// are monotone in the coordinate, so over voxel j's floats [p_j, p_j+1) the cell runs between its values at the two
// ends: c outside that range rules voxel j out exactly.
__device__ __forceinline__ unsigned sparse_axis_candidates(const SparseGeom& g, int a, float out, int cell, int kb) {
    unsigned mask = 0;
    bool exact = true;
    float p = voxel_start(kb - 1, g.v, g.inv_v, &exact);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float q = voxel_start(kb + i, g.v, g.inv_v, &exact);
        const int c0 = sparse_cell_axis(g, a, p, out), c1 = sparse_cell_axis(g, a, nextafterf(q, -INFINITY), out);
        if (!exact || (cell >= min(c0, c1) && cell <= max(c0, c1))) mask |= 1u << i;
        p = q;
    }
    return mask;
}

// one thread per (output, kernel cell): binary search of every candidate voxel, the exact predicate on the inputs
// found there, the lowest accepted id over all of them
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
    const float op[3] = {out_pos[3 * o], out_pos[3 * o + 1], out_pos[3 * o + 2]};
    int kb[3];
    unsigned cand[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float rel = ((float)cc[a] + 0.5f - g.off[a] - 0.5f * (float)g.ks[a]) * g.v;   // cell centre
        kb[a] = voxel_of(g.transpose ? op[a] - rel : op[a] + rel, g.inv_v);
        cand[a] = sparse_axis_candidates(g, a, op[a], cc[a], kb[a]);
    }
    uint32_t found = (uint32_t)n;
    for (int ix = 0; ix < 3; ++ix) {
        if (!(cand[0] >> ix & 1)) continue;
        for (int iy = 0; iy < 3; ++iy) {
            if (!(cand[1] >> iy & 1)) continue;
            for (int iz = 0; iz < 3; ++iz) {
                if (!(cand[2] >> iz & 1)) continue;
                const uint64_t key = voxel_key(kb[0] - 1 + ix, kb[1] - 1 + iy, kb[2] - 1 + iz);
                int64_t lo = 0, hi = n;
                while (lo < hi) {
                    const int64_t mid = (lo + hi) >> 1;
                    if (skeys[mid] < key) lo = mid + 1; else hi = mid;
                }
                // stable sort: ascending original id inside a key, so the first accepted input is the run's lowest
                for (int64_t j = lo; j < n && skeys[j] == key; ++j) {
                    const uint32_t id = perm[j];
                    if (id >= found) break;
                    const float* ip = in_pos + 3 * (size_t)id;
                    if (sparse_cell_axis(g, 0, ip[0], op[0]) == cx && sparse_cell_axis(g, 1, ip[1], op[1]) == cy &&
                        sparse_cell_axis(g, 2, ip[2], op[2]) == cz) {
                        found = id;
                        break;
                    }
                }
            }
        }
    }
    nbr[t] = (int32_t)found;
    if (found != (uint32_t)n && count) atomicAdd(&count[o], 1);
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
