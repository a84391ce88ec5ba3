// voxelize.cu -- hard voxelisation (hash -> stable radix sort -> segment -> emit),
// ragged_to_dense, and the fused PointPillars front end
// (pillar gather + 9-channel decoration + PFN linear/BN/ReLU/max + scatter-to-BEV).
//
// Replaces (reference call sites, /root/reference):
//   open3d.ml.torch.ops.voxelize          ml3d/torch/models/point_pillars.py:354-357
//   open3d.ml.torch.ops.ragged_to_dense   point_pillars.py:364-366, kpconv.py:2030-2032
//   PillarFeatureNet + PFNLayer           point_pillars.py:417-453, 512-555
//   PointPillarsScatter                   point_pillars.py:577-616
// Contract of the implementation-defined parts: oracle/ops_ref.c header, DESIGN.md.
//
// All of this is HBM/latency-bound integer work (12 B/point in, 8 B/point +
// 20 B/voxel out): no tensor cores here by design.
#include "../../include/o3dml_b200.h"
#include "prims.cuh"

namespace o3dml {

constexpr uint64_t VOX_INVALID_FLAG = ~0ull;

struct VoxGrid {
    float inv[3], rmin[3], rmax[3];
    int64_t ext1[3];  // extent + 1 per dim (index == extent is reachable, p == max)
    int64_t cells;    // per batch item
};

__global__ void vox_hash_kernel(const float* __restrict__ pts, int ld, int64_t n,
                                const int64_t* __restrict__ row_splits, int batch, VoxGrid g,
                                uint64_t invalid_key, uint64_t* __restrict__ keys) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    // batch id: upper bound over row_splits (batch is small)
    int lo = 0, hi = batch;  // invariant: row_splits[lo] <= i < row_splits[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (row_splits[mid] <= i) lo = mid; else hi = mid;
    }
    bool ok = i >= row_splits[0] && i < row_splits[batch];
    const float* p = pts + (size_t)i * ld;
    int64_t ijk[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float v = p[d];
        ok = ok && (v >= g.rmin[d]) && (v <= g.rmax[d]);
        ijk[d] = (int64_t)__fmul_rn(__fsub_rn(v, g.rmin[d]), g.inv[d]);
    }
    uint64_t key = invalid_key;
    if (ok) {
        key = (uint64_t)lo * (uint64_t)g.cells +
              (uint64_t)(ijk[0] + g.ext1[0] * (ijk[1] + g.ext1[1] * ijk[2]));
    }
    keys[i] = key;
}

// flags[j] = 1 for the first sorted entry of every voxel
__global__ void vox_heads_kernel(const uint64_t* __restrict__ ks, int64_t n, uint64_t invalid_key,
                                 uint32_t* __restrict__ flags, uint32_t* __restrict__ n_valid) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint64_t k = ks[j];
    bool valid = k != invalid_key;
    flags[j] = (valid && (j == 0 || ks[j - 1] != k)) ? 1u : 0u;
    if (valid && (j == n - 1 || ks[j + 1] == invalid_key)) *n_valid = (uint32_t)(j + 1);
}

__global__ void vox_headpos_kernel(const uint32_t* __restrict__ flags_excl,
                                   const uint64_t* __restrict__ ks, int64_t n,
                                   uint64_t invalid_key, uint32_t* __restrict__ head_pos) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    uint64_t k = ks[j];
    if (k != invalid_key && (j == 0 || ks[j - 1] != k)) head_pos[flags_excl[j]] = (uint32_t)j;
}

// One block.  batch_first[b] = ordinal of the first voxel of batch b (lower bound search on the
// sorted keys); batch_out[b] = first OUTPUT voxel of batch b after the max_voxels cap.
__global__ void vox_batch_bounds_kernel(const uint64_t* __restrict__ ks,
                                        const uint32_t* __restrict__ flags_excl,
                                        const uint32_t* __restrict__ m_all,
                                        const uint32_t* __restrict__ n_valid, int batch,
                                        uint64_t cells, int64_t max_voxels,
                                        uint32_t* __restrict__ batch_first,
                                        uint32_t* __restrict__ batch_out,
                                        int64_t* __restrict__ voxel_batch_splits) {
    const uint32_t nv = *n_valid;
    for (int b = threadIdx.x; b <= batch; b += blockDim.x) {
        uint64_t target = (uint64_t)b * cells;
        uint32_t lo = 0, hi = nv;  // first position with key >= target
        while (lo < hi) {
            uint32_t mid = (lo + hi) >> 1;
            if (ks[mid] < target) lo = mid + 1; else hi = mid;
        }
        batch_first[b] = (lo < nv) ? flags_excl[lo] : *m_all;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t run = 0;
        for (int b = 0; b < batch; ++b) {
            batch_out[b] = run;
            if (voxel_batch_splits) voxel_batch_splits[b] = run;
            int64_t c = (int64_t)batch_first[b + 1] - (int64_t)batch_first[b];
            run += (uint32_t)(c < max_voxels ? c : max_voxels);
        }
        batch_out[batch] = run;
        if (voxel_batch_splits) voxel_batch_splits[batch] = run;
    }
}

__device__ __forceinline__ int vox_batch_of(uint32_t v, const uint32_t* batch_first, int batch) {
    int lo = 0, hi = batch;  // batch_first[lo] <= v < batch_first[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (batch_first[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

// kept point count per (uncapped) voxel; 0 for voxels beyond max_voxels
__global__ void vox_counts_kernel(const uint32_t* __restrict__ head_pos,
                                  const uint32_t* __restrict__ m_all,
                                  const uint32_t* __restrict__ n_valid,
                                  const uint32_t* __restrict__ batch_first, int batch,
                                  int64_t max_voxels, int64_t max_points, int64_t n,
                                  uint32_t* __restrict__ kept) {
    int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const uint32_t M = *m_all;
    if (v >= M) { kept[v] = 0; return; }
    uint32_t start = head_pos[v];
    uint32_t end = (v + 1 < M) ? head_pos[v + 1] : *n_valid;
    int b = vox_batch_of((uint32_t)v, batch_first, batch);
    int64_t c = end - start;
    bool keep = (int64_t)(v - batch_first[b]) < max_voxels;
    kept[v] = keep ? (uint32_t)(c < max_points ? c : max_points) : 0u;
}

__global__ void vox_emit_voxels_kernel(const uint64_t* __restrict__ ks,
                                       const uint32_t* __restrict__ head_pos,
                                       const uint32_t* __restrict__ m_all,
                                       const uint32_t* __restrict__ kept_excl,
                                       const uint32_t* __restrict__ kept_total,
                                       const uint32_t* __restrict__ batch_first,
                                       const uint32_t* __restrict__ batch_out, int batch,
                                       int64_t max_voxels, VoxGrid g, int64_t n,
                                       int32_t* __restrict__ coords,
                                       int64_t* __restrict__ row_splits,
                                       int32_t* __restrict__ voxel_batch,
                                       int64_t* __restrict__ counts_out) {
    int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t M = *m_all;
    const uint32_t Mout = batch_out[batch];
    if (v == 0) {
        row_splits[Mout] = *kept_total;
        counts_out[0] = Mout;
        counts_out[1] = *kept_total;
    }
    if (v >= n || v >= M) return;
    int b = vox_batch_of((uint32_t)v, batch_first, batch);
    uint32_t local = (uint32_t)v - batch_first[b];
    if ((int64_t)local >= max_voxels) return;
    uint32_t ov = batch_out[b] + local;
    uint64_t cell = ks[head_pos[v]] - (uint64_t)b * (uint64_t)g.cells;
    coords[3 * (size_t)ov + 0] = (int32_t)(cell % (uint64_t)g.ext1[0]);
    coords[3 * (size_t)ov + 1] = (int32_t)((cell / (uint64_t)g.ext1[0]) % (uint64_t)g.ext1[1]);
    coords[3 * (size_t)ov + 2] = (int32_t)(cell / (uint64_t)(g.ext1[0] * g.ext1[1]));
    row_splits[ov] = kept_excl[v];
    if (voxel_batch) voxel_batch[ov] = b;
}

__global__ void vox_emit_points_kernel(const uint64_t* __restrict__ ks,
                                       const uint32_t* __restrict__ vs,
                                       const uint32_t* __restrict__ flags_excl,
                                       const uint32_t* __restrict__ head_pos,
                                       const uint32_t* __restrict__ n_valid,
                                       const uint32_t* __restrict__ kept,
                                       const uint32_t* __restrict__ kept_excl, int64_t n,
                                       int64_t* __restrict__ point_indices) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n || j >= *n_valid) return;
    uint32_t e = flags_excl[j];
    // exclusive scan of head flags: a head at j has ordinal e, a follower e - 1
    const bool is_head = (j == 0) || (ks[j - 1] != ks[j]);
    uint32_t v = is_head ? e : e - 1;
    uint32_t rank = (uint32_t)j - head_pos[v];
    if (rank < kept[v]) point_indices[(size_t)kept_excl[v] + rank] = vs[j];
}

static int vox_make_grid(const float* vs, const float* rmin, const float* rmax, VoxGrid* g) {
    g->cells = 1;
    for (int d = 0; d < 3; ++d) {
        if (!(vs[d] > 0.f)) return 1;
        volatile float iv = 1.0f / vs[d];
        volatile float span = rmax[d] - rmin[d];
        volatile float c = span * iv;
        int64_t e = (int64_t)ceilf(c);
        if (e < 1) e = 1;
        g->inv[d] = iv;
        g->rmin[d] = rmin[d];
        g->rmax[d] = rmax[d];
        g->ext1[d] = e + 1;
        if (g->cells > (int64_t)1 << 40) return 2;
        g->cells *= (e + 1);
    }
    return 0;
}

// ------------------------------------------------------------ ragged_to_dense
template <typename T>
__global__ void ragged_to_dense_kernel(const T* __restrict__ values,
                                       const int64_t* __restrict__ row_splits, int64_t rows,
                                       int64_t cols, int64_t inner, T fill, T add,
                                       T* __restrict__ out) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t total = rows * cols * inner;
    if (t >= total) return;
    int64_t e = t % inner;
    int64_t j = (t / inner) % cols;
    int64_t i = t / (inner * cols);
    int64_t s = row_splits[i], len = row_splits[i + 1] - s;
    out[t] = (j < len) ? (T)(values[(s + j) * inner + e] + add) : (T)(fill + add);
}

// ---------------------------------------------------------------- PFN fused
// One warp per pillar; lane p owns point slot p (max_num_points <= 32); every
// lane owns output channels {lane, lane+32, ...}.  Padded slots contribute the
// per-channel constant relu(BN(0)) to the max (SURVEY.md A1).
//
// TWO: the two-layer PillarFeatureNet (feat_channels [64, 64], point_pillars.py:400-453).  Wt / scale / shift are
// layer 0 ([C+5][32], lane j owns unit j) and l1 is layer 1 (input [y0[p] | m0], 64 -> COUT = 64).  Only layer 0's
// input is masked, so a padded slot's layer-1 input is [relu(BN0(0)) | m0]: its value depends on the pillar and is
// computed per pillar (SURVEY.md A13).  Layer 0 runs twice per valid slot (once for m0, once for layer 1) rather
// than keeping y0 of all slots.
struct PfnLayer1 {
    const float* w_t;    // [64][COUT] = linear.weight^T, staged in shared memory
    const float* scale;  // [COUT]
    const float* shift;  // [COUT]
};

constexpr int PFN_MAXCIN = 16;

// relu(BN0(W0 . f[p])) of this lane's layer-0 unit for slot p (the slot's decorated features live in lane p)
__device__ __forceinline__ float pfn0_unit(const float (&f)[PFN_MAXCIN], const float (&w)[PFN_MAXCIN][1], float sc,
                                           float sh, int cin, int p) {
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < PFN_MAXCIN; ++c)
        if (c < cin) acc = fmaf(__shfl_sync(0xffffffffu, f[c], p), w[c][0], acc);
    return fmaxf(fmaf(acc, sc, sh), 0.f);
}

template <int COUT, bool TWO = false>
__global__ void __launch_bounds__(256)
pp_pfn_scatter_kernel(const float* __restrict__ pts, int ld, int C,
                      const int32_t* __restrict__ coords,      // [M,3] x,y,z
                      const int64_t* __restrict__ row_splits,  // [M+1]
                      const int64_t* __restrict__ point_indices,
                      const int32_t* __restrict__ voxel_batch,  // [M] or null (batch 0)
                      const int64_t* __restrict__ num_voxels_dev, int64_t num_voxels_host,
                      const float* __restrict__ Wt,     // [C+5][COUT]   (TWO: [C+5][32])
                      const float* __restrict__ scale,  // [COUT]        (TWO: [32])
                      const float* __restrict__ shift,  // [COUT]        (TWO: [32])
                      float vx, float vy, float x_off, float y_off, int nx, int ny, int max_pts,
                      float* __restrict__ feat_out,     // [M,COUT] or null
                      float* __restrict__ canvas, int canvas_nchw, PfnLayer1 l1) {
    static_assert(!TWO || COUT == 64, "the two-layer PFN is built for 64 output channels");
    constexpr int NCH = COUT / 32;
    constexpr int NW = TWO ? 1 : NCH;  // channels per lane of the first layer
    constexpr int MAXCIN = PFN_MAXCIN;
    const int lane = threadIdx.x & 31;
    const int64_t M = num_voxels_dev ? *num_voxels_dev : num_voxels_host;
    const int cin = C + 5;
    // weights for this lane's channels, kept in registers across pillars
    float w[MAXCIN][NW], sc[NW], sh[NW];
#pragma unroll
    for (int c = 0; c < MAXCIN; ++c)
#pragma unroll
        for (int q = 0; q < NW; ++q) w[c][q] = (c < cin) ? Wt[c * (NW * 32) + q * 32 + lane] : 0.f;
#pragma unroll
    for (int q = 0; q < NW; ++q) {
        sc[q] = scale[q * 32 + lane];
        sh[q] = shift[q * 32 + lane];
    }
    __shared__ float w1s[TWO ? 64 * COUT : 1];
    float sc1[NCH], sh1[NCH];
    if constexpr (TWO) {
        for (int i = threadIdx.x; i < 64 * COUT; i += blockDim.x) w1s[i] = l1.w_t[i];
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            sc1[q] = l1.scale[q * 32 + lane];
            sh1[q] = l1.shift[q * 32 + lane];
        }
        __syncthreads();
    }
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < M; v += warps) {
        const int64_t rs0 = row_splits[v];
        const int cnt = (int)(row_splits[v + 1] - rs0);
        const int cx = coords[3 * v + 0], cy = coords[3 * v + 1];
        const bool in_grid = cx < nx && cy < ny;  // point_pillars.py:373-380
        float f[MAXCIN];
#pragma unroll
        for (int c = 0; c < MAXCIN; ++c) f[c] = 0.f;
        if (lane < cnt) {
            const float* p = pts + (size_t)point_indices[rs0 + lane] * ld;
#pragma unroll
            for (int c = 0; c < MAXCIN - 5; ++c)
                if (c < C) f[c] = p[c];
        }
        const float fc = (float)cnt;
        const float mx = __fdiv_rn(warp_sum(f[0]), fc);
        const float my = __fdiv_rn(warp_sum(f[1]), fc);
        const float mz = __fdiv_rn(warp_sum(f[2]), fc);
        if (lane < cnt) {
            const float ctr_x = __fadd_rn(__fmul_rn((float)cx, vx), x_off);
            const float ctr_y = __fadd_rn(__fmul_rn((float)cy, vy), y_off);
            // decoration order: [raw C | x-mx, y-my, z-mz | x-cx, y-cy]  (point_pillars.py:524-541)
            float dec[5] = {f[0] - mx, f[1] - my, f[2] - mz, f[0] - ctr_x, f[1] - ctr_y};
#pragma unroll
            for (int c = 0; c < MAXCIN; ++c)
#pragma unroll
                for (int e = 0; e < 5; ++e)
                    if (c == C + e) f[c] = dec[e];
        }
        float best[NCH];
        if constexpr (!TWO) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) best[q] = (cnt < max_pts) ? fmaxf(sh[q], 0.f) : 0.f;
            for (int p = 0; p < cnt; ++p) {
                float acc[NCH];
#pragma unroll
                for (int q = 0; q < NCH; ++q) acc[q] = 0.f;
#pragma unroll
                for (int c = 0; c < MAXCIN; ++c) {
                    if (c < cin) {
                        float fv = __shfl_sync(0xffffffffu, f[c], p);
#pragma unroll
                        for (int q = 0; q < NCH; ++q) acc[q] = fmaf(fv, w[c][q], acc[q]);
                    }
                }
#pragma unroll
                for (int q = 0; q < NCH; ++q)
                    best[q] = fmaxf(best[q], fmaxf(fmaf(acc[q], sc[q], sh[q]), 0.f));
            }
        } else {
            // layer 0: m0 = max over all max_pts slots, padded ones giving relu(BN0(0))
            const bool padded = cnt < max_pts;
            const float pad0 = fmaxf(sh[0], 0.f);
            float m0 = padded ? pad0 : 0.f;
            for (int p = 0; p < cnt; ++p) m0 = fmaxf(m0, pfn0_unit(f, w, sc[0], sh[0], cin, p));
            // layer 1: W1[:, 32:] . m0 is shared by every slot; the padded slot's value is the same product on
            // [relu(BN0(0)) | m0]
            float base[NCH], pad[NCH];
#pragma unroll
            for (int q = 0; q < NCH; ++q) base[q] = pad[q] = 0.f;
#pragma unroll 8
            for (int k = 0; k < 32; ++k) {
                const float mk = __shfl_sync(0xffffffffu, m0, k);
                const float pk = __shfl_sync(0xffffffffu, pad0, k);
#pragma unroll
                for (int q = 0; q < NCH; ++q) {
                    base[q] = fmaf(mk, w1s[(32 + k) * COUT + q * 32 + lane], base[q]);
                    pad[q] = fmaf(pk, w1s[k * COUT + q * 32 + lane], pad[q]);
                }
            }
#pragma unroll
            for (int q = 0; q < NCH; ++q)
                best[q] = padded ? fmaxf(fmaf(pad[q] + base[q], sc1[q], sh1[q]), 0.f) : 0.f;
            for (int p = 0; p < cnt; ++p) {
                const float y0 = pfn0_unit(f, w, sc[0], sh[0], cin, p);
                float acc[NCH];
#pragma unroll
                for (int q = 0; q < NCH; ++q) acc[q] = 0.f;
#pragma unroll 8
                for (int k = 0; k < 32; ++k) {
                    const float yk = __shfl_sync(0xffffffffu, y0, k);
#pragma unroll
                    for (int q = 0; q < NCH; ++q) acc[q] = fmaf(yk, w1s[k * COUT + q * 32 + lane], acc[q]);
                }
#pragma unroll
                for (int q = 0; q < NCH; ++q)
                    best[q] = fmaxf(best[q], fmaxf(fmaf(acc[q] + base[q], sc1[q], sh1[q]), 0.f));
            }
        }
        if (feat_out) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) feat_out[(size_t)v * COUT + q * 32 + lane] = best[q];
        }
        if (canvas && in_grid) {
            const int b = voxel_batch ? voxel_batch[v] : 0;
            if (canvas_nchw) {
                const size_t plane = (size_t)ny * nx;
#pragma unroll
                for (int q = 0; q < NCH; ++q)
                    canvas[((size_t)b * COUT + q * 32 + lane) * plane + (size_t)cy * nx + cx] = best[q];
            } else {
                float* dst = canvas + (((size_t)b * ny + cy) * nx + cx) * COUT;
#pragma unroll
                for (int q = 0; q < NCH; ++q) dst[q * 32 + lane] = best[q];
            }
        }
    }
}

struct VoxBuffers {
    RadixSortBufs sort;
    uint32_t *flags, *head_pos, *kept, *kept_excl, *batch_first, *batch_out;
    void* scan_tmp;
    uint32_t* scalars;  // [0]=n_valid [1]=m_all [2]=kept_total
};

static VoxBuffers vox_carve(Workspace& ws, int64_t n, int64_t batch) {
    VoxBuffers b;
    b.sort = radix_sort_carve(ws, n);
    b.flags = ws.take<uint32_t>(n + 1);
    b.head_pos = ws.take<uint32_t>(n + 1);
    b.kept = ws.take<uint32_t>(n + 1);
    b.kept_excl = ws.take<uint32_t>(n + 1);
    b.scan_tmp = scan_carve(ws, n + 1);
    b.batch_first = ws.take<uint32_t>(batch + 2);
    b.batch_out = ws.take<uint32_t>(batch + 2);
    b.scalars = ws.take<uint32_t>(16);
    return b;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" size_t o3dml_voxelize_workspace_bytes(int64_t n, int64_t batch) {
    return Workspace::measure(vox_carve, n, batch);
}

extern "C" int o3dml_voxelize(const float* points, int64_t num_points, int point_stride,
                              const int64_t* row_splits, int64_t batch, const float* h_voxel_size,
                              const float* h_range_min, const float* h_range_max,
                              int64_t max_points_per_voxel, int64_t max_voxels,
                              int32_t* voxel_coords, int64_t* voxel_point_indices,
                              int64_t* voxel_point_row_splits, int64_t* voxel_batch_splits,
                              int32_t* voxel_batch_id, int64_t* d_counts, void* workspace,
                              size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(num_points >= 0 && batch >= 1 && point_stride >= 3, "voxelize: bad sizes");
    O3DML_CHECK(num_points < ((int64_t)1 << 31), "voxelize: more than 2^31 points");
    O3DML_CHECK(max_points_per_voxel >= 1 && max_voxels >= 1, "voxelize: caps must be >= 1");
    VoxGrid g;
    int rc = vox_make_grid(h_voxel_size, h_range_min, h_range_max, &g);
    O3DML_CHECK(rc == 0, rc == 1 ? "voxelize: voxel_size must be positive"
                                 : "voxelize: grid too large (> 2^40 cells)");
    O3DML_CHECK((double)g.cells * (double)batch < 4.0e18, "voxelize: grid x batch too large");
    const int64_t n = num_points;
    if (n == 0) {
        O3DML_CUDA(cudaMemsetAsync(d_counts, 0, 2 * sizeof(int64_t), st));
        O3DML_CUDA(cudaMemsetAsync(voxel_point_row_splits, 0, sizeof(int64_t), st));
        if (voxel_batch_splits)
            O3DML_CUDA(cudaMemsetAsync(voxel_batch_splits, 0, (batch + 1) * sizeof(int64_t), st));
        return O3DML_OK;
    }
    Workspace ws(workspace, workspace_bytes);
    VoxBuffers b = vox_carve(ws, n, batch);
    O3DML_CHECK_WORKSPACE(ws, "voxelize");

    const uint64_t invalid_key = (uint64_t)g.cells * (uint64_t)batch;  // sorts last
    int num_bits = 1;
    while (num_bits < 64 && (invalid_key >> num_bits) != 0) ++num_bits;

    const int T = 256;
    const unsigned nb = (unsigned)ceil_div<int64_t>(n, T);
    uint32_t* scalars = b.scalars;
    O3DML_CUDA(cudaMemsetAsync(scalars, 0, 16 * sizeof(uint32_t), st));
    O3DML_CUDA(launch<vox_hash_kernel>(nb, T, 0, st, points, point_stride, n, row_splits, (int)batch, g, invalid_key,
                                       b.sort.keys_a));
    O3DML_CUDA(radix_sort_pairs(b.sort, true, n, num_bits, st));
    const uint64_t* ks = b.sort.keys_a;
    const uint32_t* vs = b.sort.vals_a;
    O3DML_CUDA(launch<vox_heads_kernel>(nb, T, 0, st, ks, n, invalid_key, b.flags, &scalars[0]));
    O3DML_CUDA(exclusive_scan_u32(b.flags, b.flags, n, &scalars[1], b.scan_tmp, st));
    O3DML_CUDA(launch<vox_headpos_kernel>(nb, T, 0, st, b.flags, ks, n, invalid_key, b.head_pos));
    O3DML_CUDA(launch<vox_batch_bounds_kernel>(1, 256, 0, st, ks, b.flags, &scalars[1], &scalars[0], (int)batch,
                                               (uint64_t)g.cells, max_voxels, b.batch_first, b.batch_out,
                                               voxel_batch_splits));
    O3DML_CUDA(launch<vox_counts_kernel>(nb, T, 0, st, b.head_pos, &scalars[1], &scalars[0], b.batch_first, (int)batch,
                                         max_voxels, max_points_per_voxel, n, b.kept));
    O3DML_CUDA(exclusive_scan_u32(b.kept, b.kept_excl, n, &scalars[2], b.scan_tmp, st));
    O3DML_CUDA(launch<vox_emit_voxels_kernel>(nb, T, 0, st, ks, b.head_pos, &scalars[1], b.kept_excl, &scalars[2],
                                              b.batch_first, b.batch_out, (int)batch, max_voxels, g, n, voxel_coords,
                                              voxel_point_row_splits, voxel_batch_id, d_counts));
    O3DML_CUDA(launch<vox_emit_points_kernel>(nb, T, 0, st, ks, vs, b.flags, b.head_pos, &scalars[0], b.kept,
                                              b.kept_excl, n, voxel_point_indices));
    return O3DML_OK;
}

extern "C" int o3dml_ragged_to_dense(const void* values, int elem_bytes, int64_t inner,
                                     const int64_t* row_splits, int64_t rows, int64_t out_col_size,
                                     int64_t fill_bits, int64_t add, void* out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(elem_bytes == 4 || elem_bytes == 8, "ragged_to_dense: 4- or 8-byte elements only");
    O3DML_CHECK(rows >= 0 && out_col_size >= 0 && inner >= 1, "ragged_to_dense: bad sizes");
    int64_t total = rows * out_col_size * inner;
    if (total == 0) return O3DML_OK;
    unsigned nb = (unsigned)ceil_div<int64_t>(total, 256);
    if (elem_bytes == 8)
        O3DML_CUDA(launch<ragged_to_dense_kernel<int64_t>>(nb, 256, 0, st, (const int64_t*)values, row_splits, rows,
                                                           out_col_size, inner, (int64_t)fill_bits, (int64_t)add,
                                                           (int64_t*)out));
    else
        O3DML_CUDA(launch<ragged_to_dense_kernel<int32_t>>(nb, 256, 0, st, (const int32_t*)values, row_splits, rows,
                                                           out_col_size, inner, (int32_t)fill_bits, (int32_t)add,
                                                           (int32_t*)out));
    return O3DML_OK;
}

// The argument checks and the launch of both PFN entries; TWO selects the two-layer kernel (l1 unused otherwise).
template <bool TWO>
static int pp_pfn_scatter_launch(const float* points, int point_stride, int point_channels,
                                 const int32_t* voxel_coords, const int64_t* voxel_row_splits,
                                 const int64_t* voxel_point_indices, const int32_t* voxel_batch_id,
                                 const int64_t* d_num_voxels, int64_t num_voxels_bound, const float* w_t,
                                 const float* bn_scale, const float* bn_shift, PfnLayer1 l1, int out_channels,
                                 float vx, float vy, float x_offset, float y_offset, int nx, int ny,
                                 int max_points_per_voxel, float* feat_out, float* canvas, int canvas_nchw,
                                 cudaStream_t st) {
    O3DML_CHECK(point_channels >= 3 && point_channels <= 11, "pfn: 3..11 point channels supported");
    O3DML_CHECK(max_points_per_voxel >= 1 && max_points_per_voxel <= 32,
                "pfn: max_points_per_voxel must be <= 32 for the fused kernel");
    O3DML_CHECK(out_channels == 64, "pfn: fused kernel is built for 64 output channels");
    if (num_voxels_bound <= 0) return O3DML_OK;
    int64_t warps_needed = num_voxels_bound;
    int64_t blocks = ceil_div<int64_t>(warps_needed, 8);
    int64_t cap = (int64_t)device_sm_count() * 8;  // 8 resident CTAs of 256 threads per SM
    if (blocks > cap) blocks = cap;
    O3DML_CUDA(launch<pp_pfn_scatter_kernel<64, TWO>>(
        (unsigned)blocks, 256, 0, st, points, point_stride, point_channels, voxel_coords, voxel_row_splits,
        voxel_point_indices, voxel_batch_id, d_num_voxels, num_voxels_bound, w_t, bn_scale, bn_shift, vx, vy, x_offset,
        y_offset, nx, ny, max_points_per_voxel, feat_out, canvas, canvas_nchw, l1));
    return O3DML_OK;
}

extern "C" int o3dml_pp_pfn_scatter(const float* points, int point_stride, int point_channels,
                                    const int32_t* voxel_coords, const int64_t* voxel_row_splits,
                                    const int64_t* voxel_point_indices, const int32_t* voxel_batch_id,
                                    const int64_t* d_num_voxels, int64_t num_voxels_bound,
                                    const float* w_t, const float* bn_scale, const float* bn_shift,
                                    int out_channels, float vx, float vy, float x_offset,
                                    float y_offset, int nx, int ny, int max_points_per_voxel,
                                    float* feat_out, float* canvas, int canvas_nchw, void* stream) {
    return pp_pfn_scatter_launch<false>(points, point_stride, point_channels, voxel_coords, voxel_row_splits,
                                        voxel_point_indices, voxel_batch_id, d_num_voxels, num_voxels_bound, w_t,
                                        bn_scale, bn_shift, PfnLayer1{}, out_channels, vx, vy, x_offset, y_offset, nx,
                                        ny, max_points_per_voxel, feat_out, canvas, canvas_nchw, (cudaStream_t)stream);
}

extern "C" int o3dml_pp_pfn2_scatter(const float* points, int point_stride, int point_channels,
                                     const int32_t* voxel_coords, const int64_t* voxel_row_splits,
                                     const int64_t* voxel_point_indices, const int32_t* voxel_batch_id,
                                     const int64_t* d_num_voxels, int64_t num_voxels_bound, const float* w0_t,
                                     const float* bn0_scale, const float* bn0_shift, const float* w1_t,
                                     const float* bn1_scale, const float* bn1_shift, int out_channels, float vx,
                                     float vy, float x_offset, float y_offset, int nx, int ny,
                                     int max_points_per_voxel, float* feat_out, float* canvas, int canvas_nchw,
                                     void* stream) {
    return pp_pfn_scatter_launch<true>(points, point_stride, point_channels, voxel_coords, voxel_row_splits,
                                       voxel_point_indices, voxel_batch_id, d_num_voxels, num_voxels_bound, w0_t,
                                       bn0_scale, bn0_shift, PfnLayer1{w1_t, bn1_scale, bn1_shift}, out_channels, vx,
                                       vy, x_offset, y_offset, nx, ny, max_points_per_voxel, feat_out, canvas,
                                       canvas_nchw, (cudaStream_t)stream);
}
