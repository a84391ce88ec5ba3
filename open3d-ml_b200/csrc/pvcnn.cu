// pvcnn.cu -- the point <-> voxel steps of PVConv (ml3d/torch/models/pvcnn.py:559-664) on channels-last grids:
// voxel coordinates and cell ids of every point, the mean of the points of every cell, trilinear devoxelization.
// Grids are [B, X, Y, Z, C] with z fastest among the spatial axes, i.e. cell (x * r + y) * r + z of cloud b is row
// b * r^3 + (x * r + y) * r + z.  Nothing here adds floats atomically: two runs agree bit for bit.
#include "../../include/o3dml_b200.h"
#include "common.cuh"

namespace o3dml {

constexpr int PV_STATS_THREADS = 1024;

// sums s[0 .. PV_STATS_THREADS) into s[0] pairwise, in an order fixed by the block size alone
__device__ __forceinline__ void block_tree_sum(float* s, int tid) {
    for (int h = PV_STATS_THREADS / 2; h > 0; h >>= 1) {
        __syncthreads();
        if (tid < h) s[tid] = __fadd_rn(s[tid], s[tid + h]);
    }
    __syncthreads();
}

// One CTA per cloud: stats[b] = (mean x, mean y, mean z, 2 * max_n |c_n - mean| + eps).  Thread t sums points
// t, t + 1024, ... in that order and the 1024 partial sums are added pairwise.
__global__ void __launch_bounds__(PV_STATS_THREADS)
pv_cloud_stats_kernel(const float* __restrict__ coords, int N, float eps, float* __restrict__ stats) {
    __shared__ float s[3][PV_STATS_THREADS];
    const int tid = threadIdx.x;
    const float* c = coords + (size_t)blockIdx.x * N * 3;
    float a[3] = {0.f, 0.f, 0.f};
    for (int n = tid; n < N; n += PV_STATS_THREADS)
#pragma unroll
        for (int d = 0; d < 3; ++d) a[d] = __fadd_rn(a[d], c[(size_t)n * 3 + d]);
    float mean[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        s[d][tid] = a[d];
        block_tree_sum(s[d], tid);
        mean[d] = __fdiv_rn(s[d][0], (float)N);
    }
    float m = 0.f;
    for (int n = tid; n < N; n += PV_STATS_THREADS) {
        const float dx = __fsub_rn(c[(size_t)n * 3], mean[0]), dy = __fsub_rn(c[(size_t)n * 3 + 1], mean[1]);
        const float dz = __fsub_rn(c[(size_t)n * 3 + 2], mean[2]);
        m = fmaxf(m, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz))));
    }
    __syncthreads();
    s[0][tid] = m;
    for (int h = PV_STATS_THREADS / 2; h > 0; h >>= 1) {
        __syncthreads();
        if (tid < h) s[0][tid] = fmaxf(s[0][tid], s[0][tid + h]);
    }
    if (tid == 0) {
        float* o = stats + (size_t)blockIdx.x * 4;
        o[0] = mean[0]; o[1] = mean[1]; o[2] = mean[2];
        o[3] = __fadd_rn(__fmul_rn(s[0][0], 2.f), eps);
    }
}

// Per point: v = clamp(((c - mean) / denom + 0.5) * r, 0, r - 1) per axis, each operation rounded on its own as the
// reference's tensor expression is, and the cell of round-half-to-even(v).
__global__ void __launch_bounds__(256)
pv_point_cells_kernel(const float* __restrict__ coords, const float* __restrict__ stats, int64_t total, int N, int r,
                      float* __restrict__ vox, int32_t* __restrict__ cell) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= total) return;
    const int b = (int)(n / N);
    const float* st = stats + (size_t)b * 4;
    int q[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float v = __fadd_rn(__fdiv_rn(__fsub_rn(coords[n * 3 + d], st[d]), st[3]), 0.5f);
        v = fminf(fmaxf(__fmul_rn(v, (float)r), 0.f), (float)(r - 1));
        vox[n * 3 + d] = v;
        q[d] = (int)rintf(v);
    }
    cell[n] = ((b * r + q[0]) * r + q[1]) * r + q[2];
}

// One thread per (cell, channel) of the dense grid: the mean, in list order, of the points grouped into the cell, zero
// for an empty cell and for the padding channels.  Every element of the grid is written.
__global__ void __launch_bounds__(256)
pv_cell_mean_kernel(const int64_t* __restrict__ splits, const int32_t* __restrict__ ids, const float* __restrict__ feat,
                    int ld, int C, int Cpad, int64_t total, float* __restrict__ grid) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int64_t cell = t / Cpad;
    const int c = (int)(t - cell * Cpad);
    float v = 0.f;
    if (c < C) {
        const int64_t a = splits[cell], e = splits[cell + 1];
        if (e > a) {
            for (int64_t i = a; i < e; ++i) v = __fadd_rn(v, feat[(size_t)ids[i] * ld + c]);
            v = __fdiv_rn(v, (float)(e - a));
        }
    }
    grid[t] = v;
}

// One warp per point.  Per axis lo = floor(v), d = v - lo, hi = lo + (d > 0): corner k takes hi on x / y / z where bit
// 2 / 1 / 0 of k is set and weighs by the product of d (hi) or 1 - d (lo).  The eight rows are added in corner order.
__global__ void __launch_bounds__(256)
pv_devoxelize_kernel(const float* __restrict__ vox, const float* __restrict__ grid, int64_t total, int N, int r, int C,
                     int grid_ld, int accumulate, float* __restrict__ out, int out_ld, int32_t* __restrict__ inds,
                     float* __restrict__ wgts) {
    const int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (n >= total) return;
    const int64_t b = n / N;
    int lo[3], step[3];
    float d[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float v = vox[n * 3 + a], f = floorf(v);
        lo[a] = (int)f;
        d[a] = __fsub_rn(v, f);
        step[a] = d[a] > 0.f ? 1 : 0;
    }
    int idx[8];
    float w[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int bx = k >> 2, by = (k >> 1) & 1, bz = k & 1;
        idx[k] = ((lo[0] + bx * step[0]) * r + lo[1] + by * step[1]) * r + lo[2] + bz * step[2];
        w[k] = __fmul_rn(__fmul_rn(bx ? d[0] : __fsub_rn(1.f, d[0]), by ? d[1] : __fsub_rn(1.f, d[1])),
                         bz ? d[2] : __fsub_rn(1.f, d[2]));
    }
    if (lane < 8) {
        const int64_t at = (b * 8 + lane) * N + (n - b * N);
        if (inds) inds[at] = idx[lane];
        if (wgts) wgts[at] = w[lane];
    }
    const float* g = grid + (size_t)b * r * r * r * grid_ld;
    float* o = out + (size_t)n * out_ld;
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) acc = fmaf(w[k], g[(size_t)idx[k] * grid_ld + c], acc);
        o[c] = accumulate ? __fadd_rn(o[c], acc) : acc;
    }
}

}  // namespace o3dml

using namespace o3dml;

extern "C" int o3dml_pv_voxel_cells(const float* coords, int batch, int num_points, int resolution, float eps,
                                    float* stats, float* voxel_coords, int32_t* cell_ids, void* stream) {
    O3DML_CHECK(coords && stats && voxel_coords && cell_ids, "pv_voxel_cells: null argument");
    O3DML_CHECK(batch > 0 && num_points > 0 && resolution > 0, "pv_voxel_cells: batch, num_points and resolution >= 1");
    const int64_t r = resolution;
    O3DML_CHECK(batch * r * r * r < ((int64_t)1 << 31), "pv_voxel_cells: 2^31 or more cells");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t total = (int64_t)batch * num_points;
    O3DML_CUDA(launch<pv_cloud_stats_kernel>(batch, PV_STATS_THREADS, 0, st, coords, num_points, eps, stats));
    O3DML_CUDA(launch<pv_point_cells_kernel>((unsigned)ceil_div<int64_t>(total, 256), 256, 0, st, coords, stats, total,
                                             num_points, resolution, voxel_coords, cell_ids));
    return O3DML_OK;
}

extern "C" int o3dml_pv_cell_mean(const int64_t* cell_row_splits, const int32_t* point_ids, int64_t num_cells,
                                  const float* features, int features_ld, int channels, int channels_pad, float* grid,
                                  void* stream) {
    O3DML_CHECK(cell_row_splits && point_ids && features && grid, "pv_cell_mean: null argument");
    O3DML_CHECK(num_cells > 0 && channels > 0 && features_ld >= channels && channels_pad >= channels,
                "pv_cell_mean: bad sizes");
    const int64_t total = num_cells * channels_pad;
    O3DML_CHECK(ceil_div<int64_t>(total, 256) < ((int64_t)1 << 31), "pv_cell_mean: grid too large");
    O3DML_CUDA(launch<pv_cell_mean_kernel>((unsigned)ceil_div<int64_t>(total, 256), 256, 0, (cudaStream_t)stream,
                                           cell_row_splits, point_ids, features, features_ld, channels, channels_pad,
                                           total, grid));
    return O3DML_OK;
}

extern "C" int o3dml_trilinear_devoxelize(const float* voxel_coords, int batch, int num_points, int resolution,
                                          const float* grid, int channels, int grid_ld, int accumulate, float* out,
                                          int out_ld, int32_t* inds, float* wgts, void* stream) {
    O3DML_CHECK(voxel_coords && grid && out, "trilinear_devoxelize: null argument");
    O3DML_CHECK(batch > 0 && num_points > 0 && resolution > 0 && channels > 0 && grid_ld >= channels &&
                    out_ld >= channels,
                "trilinear_devoxelize: bad sizes");
    const int64_t total = (int64_t)batch * num_points;
    O3DML_CUDA(launch<pv_devoxelize_kernel>((unsigned)ceil_div<int64_t>(total, 8), 256, 0, (cudaStream_t)stream,
                                            voxel_coords, grid, total, num_points, resolution, channels, grid_ld,
                                            accumulate, out, out_ld, inds, wgts));
    return O3DML_OK;
}
