// grid.cu -- uniform hash-grid neighbour search: exact k-NN and fixed-radius search,
// batched through row_splits.  Support points are counting-sorted into cells and
// stored as float4 (x, y, z, original index) so that every candidate is one
// coalesced 16-byte load; queries are processed in cell order so that the lanes
// of a warp walk the same cells.
//
// Replaces (reference call sites, /root/reference):
//   open3d.core.nns.NearestNeighborSearch.knn_search   ml3d/datasets/utils/dataprocessing.py:99-103
//                                                      (<- RandLANet.transform randlanet.py:218-229)
//   open3d.ml.torch.ops.knn_search                     ml3d/torch/models/point_transformer.py:724-734
//   open3d.ml.torch.layers.FixedRadiusSearch           ml3d/torch/models/kpconv.py:2021-2026
//   open3d.ml.torch.ops.radius_search / layers.RadiusSearch (no call site; DESIGN.md section 2)
// Result order (implementation-defined upstream, fixed here): rows ascend by
// (distance, index); in float32 without FMA, d = q - p per axis, L2 is returned squared,
// ((dx*dx + dy*dy) + dz*dz), L1 is (|dx| + |dy|) + |dz| and Linf max(max(|dx|, |dy|), |dz|)
// (oracle/ops_ref.c, oracle/search_ref.c).  Non-finite input: a NaN distance (a NaN coordinate, or +inf - +inf) is
// never ranked nor within a radius; a distance that is +inf (an infinite coordinate, or an overflowing sum) ranks
// after every finite one; so a k-NN row may be short, padded with -1 / +inf.  An axis whose bounding-box extent is
// not finite gets one cell (grid_setup_kernel): the search stays exact, at the cost of visiting more points.
// HBM/latency-bound: 12 B/query in, 8*k (or 4*L) B/query out.
#include "../../include/o3dml_b200.h"
#include "prims.cuh"
#include <float.h>

namespace o3dml {

struct GridInfo {       // one per batch item, device resident
    float ox, oy, oz;   // origin (bbox min)
    float cs, inv_cs;   // cell size
    int dx, dy, dz;     // grid dims
    uint32_t cell_base; // first cell of this batch item in the global cell arrays
    uint32_t pad;
};

__device__ __forceinline__ unsigned f2ord(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ int batch_of(int64_t i, const int64_t* splits, int batch) {
    int lo = 0, hi = batch;
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (splits[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// bbox[b][0..2] = ordered-uint min, [3..5] = ordered-uint max (initialised by grid_init_kernel)
__global__ void grid_init_kernel(unsigned* bbox, int batch) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < batch * 6) bbox[i] = (i % 6 < 3) ? 0xffffffffu : 0u;
}

__global__ void grid_bbox_kernel(const float* __restrict__ pts, int64_t n,
                                 const int64_t* __restrict__ splits, int batch, unsigned* bbox) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int b = batch_of(i, splits, batch);
    // warp-aggregate when the whole warp is in the same batch item
    float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    unsigned act = __activemask();
    int b0 = __shfl_sync(act, b, __ffs(act) - 1);
    if (__all_sync(act, b == b0) && act == 0xffffffffu) {
        float mnx = x, mny = y, mnz = z, mxx = x, mxy = y, mxz = z;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mnx = fminf(mnx, __shfl_xor_sync(0xffffffffu, mnx, o));
            mny = fminf(mny, __shfl_xor_sync(0xffffffffu, mny, o));
            mnz = fminf(mnz, __shfl_xor_sync(0xffffffffu, mnz, o));
            mxx = fmaxf(mxx, __shfl_xor_sync(0xffffffffu, mxx, o));
            mxy = fmaxf(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
            mxz = fmaxf(mxz, __shfl_xor_sync(0xffffffffu, mxz, o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&bbox[b * 6 + 0], f2ord(mnx)); atomicMin(&bbox[b * 6 + 1], f2ord(mny));
            atomicMin(&bbox[b * 6 + 2], f2ord(mnz)); atomicMax(&bbox[b * 6 + 3], f2ord(mxx));
            atomicMax(&bbox[b * 6 + 4], f2ord(mxy)); atomicMax(&bbox[b * 6 + 5], f2ord(mxz));
        }
    } else {
        atomicMin(&bbox[b * 6 + 0], f2ord(x)); atomicMin(&bbox[b * 6 + 1], f2ord(y));
        atomicMin(&bbox[b * 6 + 2], f2ord(z)); atomicMax(&bbox[b * 6 + 3], f2ord(x));
        atomicMax(&bbox[b * 6 + 4], f2ord(y)); atomicMax(&bbox[b * 6 + 5], f2ord(z));
    }
}

// cells grid_setup_kernel allows a batch item of nb points: the host sizes the cell arrays from it, without a sync
__host__ __device__ inline double grid_cell_cap(int64_t nb) { return 2.0 * (double)nb + 64.0; }

// Cell size of each batch item of a search with one radius per query: the largest valid (finite, >= 0) radius among
// the item's queries.  For r >= +0 the order of the floats is the order of their bit patterns, so a uint atomicMax
// finds it; the buffer starts at 0 = +0.0f, which an item without a valid radius keeps.
__global__ void item_radius_kernel(const float* __restrict__ radii, int64_t nq, const int64_t* __restrict__ qsplits,
                                   int batch, unsigned* __restrict__ item_radius) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const float r = radii[i];
    if (r >= 0.f && r <= FLT_MAX) atomicMax(&item_radius[batch_of(i, qsplits, batch)], __float_as_uint(fabsf(r)));
}

// One thread per batch item picks the cell size.  item_radius (per-query radii): the item's largest valid radius,
// at least 1e-6; fixed_cs > 0: radius search (cs = radius); otherwise the k-NN heuristic: the radius expected to hold
// k points at the mean surface / volume density of the bounding box.  The cell size is then raised to 2^-20 of the
// longest side of the bounding box, so that the growth below (1.26^64 > 2^21) always ends inside grid_cell_cap, and
// grows until the item's cells fit grid_cell_cap.  The cell size affects speed only: every search is exact.
// An axis whose extent is not a finite float (a NaN or infinite coordinate, or max - min past FLT_MAX) gets one cell
// and origin 0: every point and query is clamped into it, which keeps the searches exact, and no NaN or infinity
// reaches the float -> int conversions of the grid dims.
__global__ void grid_setup_kernel(const unsigned* __restrict__ bbox,
                                  const int64_t* __restrict__ splits, int batch, float fixed_cs,
                                  int k, GridInfo* __restrict__ info, uint32_t* total_cells,
                                  const unsigned* __restrict__ item_radius) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    uint32_t base = 0;
    for (int b = 0; b < batch; ++b) {
        int64_t nb = splits[b + 1] - splits[b];
        GridInfo g;
        if (nb <= 0) {
            g.ox = g.oy = g.oz = 0.f; g.cs = 1.f; g.inv_cs = 1.f; g.dx = g.dy = g.dz = 1;
        } else {
            float mn[3], mx[3], e[3];
            for (int d = 0; d < 3; ++d) {
                mn[d] = ord2f(bbox[b * 6 + d]);
                mx[d] = ord2f(bbox[b * 6 + 3 + d]);
                const float ext = mx[d] - mn[d];
                if (ext <= FLT_MAX) e[d] = fmaxf(ext, 1e-6f);
                else { e[d] = 0.f; mn[d] = 0.f; }  // NaN or infinite: one cell along this axis
            }
            float cs = item_radius ? fmaxf(__uint_as_float(item_radius[b]), 1e-6f) : fixed_cs;
            if (!(cs > 0.f)) {
                float e0 = fmaxf(e[0], fmaxf(e[1], e[2]));
                float e2 = fminf(e[0], fminf(e[1], e[2]));
                float e1 = e[0] + e[1] + e[2] - e0 - e2;
                float kk = (float)(k < 4 ? 4 : k);
                float cs2 = sqrtf(kk * e0 * e1 / (3.14159265f * (float)nb));
                float cs3 = cbrtf(kk * e0 * e1 * e2 / (4.18879f * (float)nb));
                cs = fmaxf(fmaxf(cs2, cs3), 1e-6f);
            }
            cs = fmaxf(cs, fmaxf(e[0], fmaxf(e[1], e[2])) * 0x1p-20f);
            const double cap = grid_cell_cap(nb);
            for (int it = 0; it < 64; ++it) {
                double c = (floor((double)e[0] / cs) + 1) * (floor((double)e[1] / cs) + 1) *
                           (floor((double)e[2] / cs) + 1);
                if (c <= cap) break;
                cs *= 1.26f;
            }
            g.ox = mn[0]; g.oy = mn[1]; g.oz = mn[2];
            g.cs = cs; g.inv_cs = 1.0f / cs;
            g.dx = (int)floor((double)e[0] / cs) + 1;  // same arithmetic as the cap check above
            g.dy = (int)floor((double)e[1] / cs) + 1;
            g.dz = (int)floor((double)e[2] / cs) + 1;
        }
        g.cell_base = base;
        g.pad = 0;
        info[b] = g;
        base += (uint32_t)(g.dx * g.dy * g.dz);
    }
    *total_cells = base;
}

__device__ __forceinline__ void cell_coords(const GridInfo& g, float x, float y, float z, int& cx,
                                            int& cy, int& cz) {
    cx = min(max((int)floorf((x - g.ox) * g.inv_cs), 0), g.dx - 1);
    cy = min(max((int)floorf((y - g.oy) * g.inv_cs), 0), g.dy - 1);
    cz = min(max((int)floorf((z - g.oz) * g.inv_cs), 0), g.dz - 1);
}
__device__ __forceinline__ uint32_t cell_id(const GridInfo& g, int cx, int cy, int cz) {
    return g.cell_base + (uint32_t)((cz * g.dy + cy) * g.dx + cx);
}

__global__ void grid_count_kernel(const float* __restrict__ pts, int64_t n,
                                  const int64_t* __restrict__ splits, int batch,
                                  const GridInfo* __restrict__ info, uint32_t* __restrict__ cell_of,
                                  uint32_t* __restrict__ cell_count) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int b = batch_of(i, splits, batch);
    GridInfo g = info[b];
    int cx, cy, cz;
    cell_coords(g, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], cx, cy, cz);
    uint32_t c = cell_id(g, cx, cy, cz);
    cell_of[i] = c;
    atomicAdd(&cell_count[c], 1u);
}

__global__ void grid_fill_kernel(const float* __restrict__ pts, int64_t n,
                                 const uint32_t* __restrict__ cell_of,
                                 const uint32_t* __restrict__ cell_start,
                                 uint32_t* __restrict__ cursor, float4* __restrict__ sorted) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t c = cell_of[i];
    uint32_t pos = cell_start[c] + atomicAdd(&cursor[c], 1u);
    sorted[pos] = make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], __int_as_float((int)i));
}

// Order in which queries are processed: sort query ids by the support-grid cell they fall in
// (counting sort with atomics; order inside a cell is irrelevant).
__global__ void query_cell_kernel(const float* __restrict__ q, int64_t nq,
                                  const int64_t* __restrict__ qsplits, int batch,
                                  const GridInfo* __restrict__ info, uint32_t* __restrict__ qcell,
                                  uint32_t* __restrict__ qcount) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    int b = batch_of(i, qsplits, batch);
    GridInfo g = info[b];
    int cx, cy, cz;
    cell_coords(g, q[3 * i], q[3 * i + 1], q[3 * i + 2], cx, cy, cz);
    uint32_t c = cell_id(g, cx, cy, cz);
    qcell[i] = c;
    atomicAdd(&qcount[c], 1u);
}
__global__ void query_order_kernel(int64_t nq, const uint32_t* __restrict__ qcell,
                                   const uint32_t* __restrict__ qstart,
                                   uint32_t* __restrict__ qcursor, uint32_t* __restrict__ order) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    uint32_t c = qcell[i];
    order[qstart[c] + atomicAdd(&qcursor[c], 1u)] = (uint32_t)i;
}

__device__ __forceinline__ bool nb_less(float da, int ia, float db, int ib) {
    return da < db || (da == db && ia < ib);
}

enum { L2 = O3DML_METRIC_L2, L1 = O3DML_METRIC_L1, LINF = O3DML_METRIC_LINF };

__device__ __forceinline__ float fmax_nan(float a, float b) {  // NaN if either is NaN (fmaxf would drop it)
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// The distance of metric M with the operation order of the op contract.  A NaN difference gives NaN in every
// metric, so such a point is never within a threshold nor ranked.
template <int M>
__device__ __forceinline__ float metric_dist(float qx, float qy, float qz, float px, float py, float pz) {
    if (M == L2) return sqdist3(qx, qy, qz, px, py, pz);
    const float ax = fabsf(__fsub_rn(qx, px)), ay = fabsf(__fsub_rn(qy, py)), az = fabsf(__fsub_rn(qz, pz));
    if (M == L1) return __fadd_rn(__fadd_rn(ax, ay), az);
    return fmax_nan(fmax_nan(ax, ay), az);
}

// ignore_query_point: the support point coincides with the query (== per coordinate: -0 == +0, NaN never)
__device__ __forceinline__ bool coincident(float qx, float qy, float qz, const float4& p) {
    return qx == p.x && qy == p.y && qz == p.z;
}

// ------------------------------------------------------------------- k-NN ----
// A row holds the first k points by (d, id) among those with a distance that is not NaN (+inf ranks after every finite
// distance), then -1 / +inf padding: it is short when its item holds fewer than k such points.
// IGNORE: row_len[qi] = the neighbours found (fewer than k when coincident points were skipped or the row is short).
// Without IGNORE the row stays dense [k], padded in place.
// The min-blocks hint of 1 lets ptxas give the metric / ignore instances the registers they need without spilling;
// the L2 instances keep the bare bound (0 = none), which they were tuned under.
template <int KMAX, int M = L2, bool IGNORE = false>
__global__ void __launch_bounds__(128, (M != L2 || IGNORE) ? 1 : 0)
knn_kernel(const float* __restrict__ queries, int64_t nq, const int64_t* __restrict__ qsplits,
           const int64_t* __restrict__ psplits, int batch, const uint32_t* __restrict__ order,
           const GridInfo* __restrict__ info, const uint32_t* __restrict__ cell_start,
           const float4* __restrict__ sorted, int k, void* __restrict__ out_idx, int idx_is64,
           float* __restrict__ out_d2, uint32_t* __restrict__ row_len) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq) return;
    const int64_t qi = order ? (int64_t)order[t] : t;
    const int b = batch_of(qi, qsplits, batch);
    const GridInfo g = info[b];
    const float qx = queries[3 * qi], qy = queries[3 * qi + 1], qz = queries[3 * qi + 2];
    float bd[KMAX];
    int bi[KMAX];
    const float inf = __int_as_float(0x7f800000);
#pragma unroll
    for (int j = 0; j < KMAX; ++j) { bd[j] = inf; bi[j] = 0x7fffffff; }  // empty: ranks after every point
    const int64_t nsup = psplits[b + 1] - psplits[b];
    const int kk = (int)(nsup < k ? nsup : k);  // neighbours that exist
    if (kk > 0) {
        int cx, cy, cz;
        cell_coords(g, qx, qy, qz, cx, cy, cz);
        const int rmax = max(max(max(cx, g.dx - 1 - cx), max(cy, g.dy - 1 - cy)), max(cz, g.dz - 1 - cz));
        for (int r = 0; r <= rmax; ++r) {
            const int z0 = max(cz - r, 0), z1 = min(cz + r, g.dz - 1);
            const int y0 = max(cy - r, 0), y1 = min(cy + r, g.dy - 1);
            for (int z = z0; z <= z1; ++z) {
                const bool zface = (z == cz - r) || (z == cz + r);
                for (int y = y0; y <= y1; ++y) {
                    const bool face = zface || (y == cy - r) || (y == cy + r);
                    // on a face row walk every x, otherwise only the two x-caps of the shell
                    const int xs = face ? 1 : max(2 * r, 1);
                    for (int x = cx - r; x <= cx + r; x += xs) {
                        if (x < 0 || x >= g.dx) continue;
                        const uint32_t c = cell_id(g, x, y, z);
                        const uint32_t s = cell_start[c], e = cell_start[c + 1];
                        for (uint32_t pi = s; pi < e; ++pi) {
                            const float4 pt = sorted[pi];
                            if (IGNORE && coincident(qx, qy, qz, pt)) continue;
                            const float d = metric_dist<M>(qx, qy, qz, pt.x, pt.y, pt.z);
                            const int id = __float_as_int(pt.w);
                            if (nb_less(d, id, bd[KMAX - 1], bi[KMAX - 1])) {
                                // replace the current worst (slot KMAX-1 holds the worst because
                                // unused slots are +inf) and bubble it up
                                bd[KMAX - 1] = d;
                                bi[KMAX - 1] = id;
#pragma unroll
                                for (int j = KMAX - 1; j > 0; --j) {
                                    if (nb_less(bd[j], bi[j], bd[j - 1], bi[j - 1])) {
                                        float td = bd[j]; bd[j] = bd[j - 1]; bd[j - 1] = td;
                                        int ti = bi[j]; bi[j] = bi[j - 1]; bi[j - 1] = ti;
                                    }
                                }
                            }
                        }
                    }
                }
            }
            // everything closer than r*cs has been seen (cells are >= cs wide, the query sits
            // inside its own cell or outside the grid on the far side); 1e-4 relative slack
            // covers the float rounding of the cell assignment.  That bound is in Linf, and L1 >= Linf.
            // A k-th best at +inf (or an empty slot) never stops the walk: a point further out may tie it at +inf and
            // rank first by index.
            const float cover = (float)r * g.cs * 0.9999f;
            float kth = inf;  // the k-th best so far sits at slot kk-1 (slots are sorted)
#pragma unroll
            for (int j = 0; j < KMAX; ++j)
                if (j == kk - 1) kth = bd[j];
            if (kth < inf && kth <= (M == L2 ? cover * cover : cover)) break;
        }
    }
    uint32_t found = 0;
#pragma unroll
    for (int j = 0; j < KMAX; ++j) {
        if (j < k) {
            const bool have = j < kk && bi[j] != 0x7fffffff;  // filled: NaN distances are never ranked
            if (idx_is64) ((int64_t*)out_idx)[qi * k + j] = have ? (int64_t)bi[j] : -1;
            else ((int32_t*)out_idx)[qi * k + j] = have ? bi[j] : -1;
            if (out_d2) out_d2[qi * k + j] = have ? bd[j] : __int_as_float(0x7f800000);
            found += have;
        }
    }
    if (IGNORE) row_len[qi] = found;
}

// Moves the rows of a dense [nq, k] k-NN result (row qi: row_len[qi] neighbours, then padding) to their ragged places
// row_start[qi] (the exclusive scan of row_len) of the caller's outputs.
__global__ void knn_compact_kernel(const int32_t* __restrict__ idx, const float* __restrict__ dist, int64_t nq, int k,
                                   const uint32_t* __restrict__ row_len, const uint32_t* __restrict__ row_start,
                                   void* __restrict__ out_idx, int idx_is64, float* __restrict__ out_dist) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq * k) return;
    const int64_t qi = t / k;
    const int j = (int)(t - qi * k);
    if (j >= (int)row_len[qi]) return;
    const int64_t o = (int64_t)row_start[qi] + j;
    if (idx_is64) ((int64_t*)out_idx)[o] = idx[t];
    else ((int32_t*)out_idx)[o] = idx[t];
    if (out_dist) out_dist[o] = dist[t];
}

// ----------------------------------------------------------- fixed radius ----
// inserts (d, id) into the sorted row [row, j) and keeps it sorted by (d, id)
template <typename I>
__device__ __forceinline__ void row_insert(I* idx, float* dist, int64_t row, int64_t j,
                                           float d, int id) {
    while (j > row && nb_less(d, id, dist[j - 1], (int)idx[j - 1])) {
        idx[j] = idx[j - 1];
        dist[j] = dist[j - 1];
        --j;
    }
    idx[j] = (I)id;
    dist[j] = d;
}

// mode 0: count -> counts[qi]; mode 1: fill rows at row_splits[qi], kept sorted by (d, idx).
// Without GENERAL: L2, one radius, int32 ids (o3dml_radius_count / _fill).  GENERAL: the radius of query qi is
// radii[qi] when radii is given (a negative, NaN or infinite one gives an empty row), the ids go to out_idx64 instead
// of out_idx when it is given, and with `normalize` the returned distances are divided by the threshold's scale (r * r
// for L2, r otherwise).
// GENERAL instances take the min-blocks hint of 1 for the reason given at knn_kernel.
template <int MODE, int M = L2, bool IGNORE = false, bool GENERAL = false>
__global__ void __launch_bounds__(128, GENERAL ? 1 : 0)
radius_kernel(const float* __restrict__ queries, int64_t nq, const int64_t* __restrict__ qsplits,
              int batch, const uint32_t* __restrict__ order, const GridInfo* __restrict__ info,
              const uint32_t* __restrict__ cell_start, const float4* __restrict__ sorted,
              float radius, uint32_t* __restrict__ counts, const int64_t* __restrict__ row_splits,
              int32_t* __restrict__ out_idx, float* __restrict__ out_d2, const float* __restrict__ radii,
              int64_t* __restrict__ out_idx64, int normalize) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq) return;
    const int64_t qi = order ? (int64_t)order[t] : t;
    const int b = batch_of(qi, qsplits, batch);
    const GridInfo g = info[b];
    const float qx = queries[3 * qi], qy = queries[3 * qi + 1], qz = queries[3 * qi + 2];
    if (GENERAL && radii) radius = radii[qi];
    const float r2 = M == L2 ? __fmul_rn(radius, radius) : radius;  // the threshold: d <= r2
    // cell box that contains the ball, with slack for the float cell assignment
    const float rr = radius * 1.0001f + 1e-7f;
    int x0 = (int)floorf((qx - rr - g.ox) * g.inv_cs), x1 = (int)floorf((qx + rr - g.ox) * g.inv_cs);
    int y0 = (int)floorf((qy - rr - g.oy) * g.inv_cs), y1 = (int)floorf((qy + rr - g.oy) * g.inv_cs);
    int z0 = (int)floorf((qz - rr - g.oz) * g.inv_cs), z1 = (int)floorf((qz + rr - g.oz) * g.inv_cs);
    // points are clamped into the grid when binned, so clamp the box the same way
    x0 = min(max(x0, 0), g.dx - 1); x1 = min(max(x1, 0), g.dx - 1);
    y0 = min(max(y0, 0), g.dy - 1); y1 = min(max(y1, 0), g.dy - 1);
    z0 = min(max(z0, 0), g.dz - 1); z1 = min(max(z1, 0), g.dz - 1);
    if (GENERAL && !(radius >= 0.f && radius <= FLT_MAX)) z1 = -1;  // no valid radius: visit nothing
    uint32_t cnt = 0;
    int64_t row = 0, cap = 0;
    if (MODE == 1) { row = row_splits[qi]; cap = row_splits[qi + 1] - row; }
    for (int z = z0; z <= z1; ++z)
        for (int y = y0; y <= y1; ++y) {
            const uint32_t c0 = cell_id(g, x0, y, z);
            const uint32_t s = cell_start[c0], e = cell_start[c0 + (uint32_t)(x1 - x0) + 1];
            for (uint32_t pi = s; pi < e; ++pi) {  // x-adjacent cells are contiguous
                const float4 pt = sorted[pi];
                if (IGNORE && coincident(qx, qy, qz, pt)) continue;
                const float d = metric_dist<M>(qx, qy, qz, pt.x, pt.y, pt.z);
                if (d <= r2) {
                    if (MODE == 1 && (int64_t)cnt < cap) {  // insertion keeps the row sorted
                        const int id = __float_as_int(pt.w);
                        if (GENERAL && out_idx64) row_insert(out_idx64, out_d2, row, row + cnt, d, id);
                        else row_insert(out_idx, out_d2, row, row + cnt, d, id);
                    }
                    ++cnt;
                }
            }
        }
    if (MODE == 0) counts[qi] = cnt;
    if (GENERAL && MODE == 1 && normalize) {
        const float scale = M == L2 ? r2 : radius;
        const int64_t end = row + min((int64_t)cnt, cap);
        for (int64_t j = row; j < end; ++j) out_d2[j] = __fdiv_rn(out_d2[j], scale);
    }
}

__global__ void widen_splits_kernel(const uint32_t* __restrict__ excl, int64_t n,
                                    const uint32_t* __restrict__ total,
                                    int64_t* __restrict__ out, int64_t* __restrict__ total64) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = excl[i];
    if (i == 0) { out[n] = *total; if (total64) *total64 = *total; }
}

struct GridBuf {
    unsigned* bbox; GridInfo* info; uint32_t* total_cells;
    uint32_t *cell_of, *cell_start, *cursor; float4* sorted;
    uint32_t *qcell, *qstart, *qcursor, *order;
    void* scan_tmp;
    int64_t max_cells;
};

// cells of a whole batch: the items' caps add up to 2*np + 64*batch, plus a margin of one cap(0) per item and one more
static int64_t grid_max_cells(int64_t np, int64_t batch) {
    return (int64_t)grid_cell_cap(np) + 2 * batch * (int64_t)grid_cell_cap(0);
}

static GridBuf grid_carve(Workspace& ws, int64_t np, int64_t nq, int64_t batch) {
    GridBuf g;
    g.max_cells = grid_max_cells(np, batch);
    g.bbox = ws.take<unsigned>(batch * 6);
    g.info = ws.take<GridInfo>(batch);
    g.total_cells = ws.take<uint32_t>(16);
    g.cell_of = ws.take<uint32_t>(np);
    g.cell_start = ws.take<uint32_t>(g.max_cells + 1);
    g.cursor = ws.take<uint32_t>(g.max_cells + 1);
    g.sorted = ws.take<float4>(np);
    g.qcell = ws.take<uint32_t>(nq);
    g.qstart = ws.take<uint32_t>(g.max_cells + 1);
    g.qcursor = ws.take<uint32_t>(g.max_cells + 1);
    g.order = ws.take<uint32_t>(nq);
    g.scan_tmp = scan_carve(ws, g.max_cells + 1);
    return g;
}


// Layout of the radius searches: the grid that the count entry builds and the fill entry reads back, then the
// per-query counts and their scan, then the per-item radius of a search with one radius per query.  Both entries
// carve it, so that fill finds the grid where count left it.
struct RadiusBuf : GridBuf {
    uint32_t *counts, *total;
    void* count_scan_tmp;
    unsigned* item_radius;
};

static RadiusBuf radius_carve(Workspace& ws, int64_t np, int64_t nq, int64_t batch) {
    RadiusBuf r{grid_carve(ws, np, nq, batch)};
    r.counts = ws.take<uint32_t>(nq + 1);
    r.count_scan_tmp = scan_carve(ws, nq + 1);
    r.total = ws.take<uint32_t>(16);
    r.item_radius = ws.take<unsigned>(batch);
    return r;
}

// Layout of the k-NN search: the grid and, when ignore_query_point can leave rows short, the dense rows, their lengths
// and the scan that places them.
struct KnnBuf : GridBuf {
    int32_t* idx;
    float* dist;
    uint32_t *len, *start, *total;
    void* len_scan_tmp;
};

static KnnBuf knn_carve(Workspace& ws, int64_t np, int64_t nq, int64_t batch, int k, int ragged) {
    KnnBuf b{grid_carve(ws, np, nq, batch)};
    if (ragged) {
        b.idx = ws.take<int32_t>(nq * k);
        b.dist = ws.take<float>(nq * k);
        b.len = ws.take<uint32_t>(nq);
        b.start = ws.take<uint32_t>(nq);
        b.total = ws.take<uint32_t>(16);
        b.len_scan_tmp = scan_carve(ws, nq);
    }
    return b;
}

// builds the support grid and the cell-ordered query permutation
static int grid_build(const float* pts, int64_t np, const int64_t* psplits, const float* q,
                      int64_t nq, const int64_t* qsplits, int batch, float fixed_cs, int k,
                      const unsigned* item_radius, const GridBuf& g, cudaStream_t st) {
    const int T = 256;
    const unsigned pb = (unsigned)ceil_div<int64_t>(np, T);
    O3DML_CUDA(launch<grid_init_kernel>(ceil_div(batch * 6, T), T, 0, st, g.bbox, batch));
    if (np > 0) O3DML_CUDA(launch<grid_bbox_kernel>(pb, T, 0, st, pts, np, psplits, batch, g.bbox));
    O3DML_CUDA(launch<grid_setup_kernel>(1, 32, 0, st, g.bbox, psplits, batch, fixed_cs, k, g.info, g.total_cells,
                                         item_radius));
    O3DML_CUDA(cudaMemsetAsync(g.cell_start, 0, (g.max_cells + 1) * 4, st));
    O3DML_CUDA(cudaMemsetAsync(g.cursor, 0, (g.max_cells + 1) * 4, st));
    if (np > 0)
        O3DML_CUDA(launch<grid_count_kernel>(pb, T, 0, st, pts, np, psplits, batch, g.info, g.cell_of, g.cell_start));
    O3DML_CUDA(exclusive_scan_u32(g.cell_start, g.cell_start, g.max_cells + 1, nullptr, g.scan_tmp, st));
    if (np > 0)
        O3DML_CUDA(launch<grid_fill_kernel>(pb, T, 0, st, pts, np, g.cell_of, g.cell_start, g.cursor, g.sorted));
    if (nq > 0) {
        const unsigned qb = (unsigned)ceil_div<int64_t>(nq, T);
        O3DML_CUDA(cudaMemsetAsync(g.qstart, 0, (g.max_cells + 1) * 4, st));
        O3DML_CUDA(cudaMemsetAsync(g.qcursor, 0, (g.max_cells + 1) * 4, st));
        O3DML_CUDA(launch<query_cell_kernel>(qb, T, 0, st, q, nq, qsplits, batch, g.info, g.qcell, g.qstart));
        O3DML_CUDA(exclusive_scan_u32(g.qstart, g.qstart, g.max_cells + 1, nullptr, g.scan_tmp, st));
        O3DML_CUDA(launch<query_order_kernel>(qb, T, 0, st, nq, g.qcell, g.qstart, g.qcursor, g.order));
    }
    return O3DML_OK;
}

// one radius_kernel<MODE, ...> launch: the L2 / one-radius / int32 instance unless `general`, else the instance of
// (metric, ignore_query_point)
template <int MODE, class... Args>
static cudaError_t radius_launch(bool general, int metric, int ignore, unsigned nb, cudaStream_t st, Args... args) {
    if (!general) return launch<radius_kernel<MODE>>(nb, 128, 0, st, args...);
#define RADIUS_LAUNCH(M, IG) \
    if (metric == M && !!ignore == IG) return launch<radius_kernel<MODE, M, IG, true>>(nb, 128, 0, st, args...)
    RADIUS_LAUNCH(L2, false); RADIUS_LAUNCH(L2, true);
    RADIUS_LAUNCH(L1, false); RADIUS_LAUNCH(L1, true);
    RADIUS_LAUNCH(LINF, false); RADIUS_LAUNCH(LINF, true);
#undef RADIUS_LAUNCH
    return cudaErrorInvalidValue;  // unreachable: the entries check the metric
}

// one knn_kernel<KMAX, M, IG> launch, KMAX the smallest instance that holds k
template <int M, bool IG, class... Args>
static cudaError_t knn_launch(int k, unsigned nb, cudaStream_t st, Args... args) {
    if (k == 1) return launch<knn_kernel<1, M, IG>>(nb, 128, 0, st, args...);
    if (k <= 8) return launch<knn_kernel<8, M, IG>>(nb, 128, 0, st, args...);
    if (k <= 16) return launch<knn_kernel<16, M, IG>>(nb, 128, 0, st, args...);
    if (k <= 32) return launch<knn_kernel<32, M, IG>>(nb, 128, 0, st, args...);
    return launch<knn_kernel<64, M, IG>>(nb, 128, 0, st, args...);
}

// The k-NN search of every entry.  Without ignore_query_point the rows go straight to out_index / out_distance2
// [num_queries, k]; with it they go to the workspace, and knn_compact_kernel moves them to their ragged places.
static int knn_impl(const char* name, const float* points, int64_t num_points, const int64_t* points_row_splits,
                    const float* queries, int64_t num_queries, const int64_t* queries_row_splits, int64_t batch, int k,
                    int metric, int ignore, void* out_index, int index_is64, float* out_distance2,
                    int64_t* out_row_splits, int64_t* d_total, void* workspace, size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(k >= 1 && k <= 64, "%s: k must be in 1..64 (got %d)", name, k);
    O3DML_CHECK(batch >= 1 && num_points >= 0 && num_queries >= 0, "%s: bad sizes", name);
    O3DML_CHECK(num_points < ((int64_t)1 << 30), "%s: too many points", name);
    O3DML_CHECK(metric == L2 || metric == L1 || metric == LINF, "%s: unknown metric %d", name, metric);
    if (num_queries == 0) {
        if (ignore) {
            O3DML_CUDA(cudaMemsetAsync(out_row_splits, 0, sizeof(int64_t), st));
            if (d_total) O3DML_CUDA(cudaMemsetAsync(d_total, 0, sizeof(int64_t), st));
        }
        return O3DML_OK;
    }
    Workspace ws(workspace, workspace_bytes);
    const KnnBuf g = knn_carve(ws, num_points, num_queries, batch, k, ignore);
    if (!ws.ok) O3DML_FAIL(O3DML_ERR_WORKSPACE, "%s: workspace too small (%zu needed)", name, ws.off);
    int rc = grid_build(points, num_points, points_row_splits, queries, num_queries, queries_row_splits, (int)batch,
                        0.f, k, nullptr, g, st);
    if (rc) return rc;
    const unsigned nb = (unsigned)ceil_div<int64_t>(num_queries, 128);
#define KNN_ARGS(IDX, IS64, DIST, LEN)                                                                              \
    nb, st, queries, num_queries, queries_row_splits, points_row_splits, (int)batch, g.order, g.info, g.cell_start, \
        g.sorted, k, IDX, IS64, DIST, LEN
    if (!ignore) {
        uint32_t* no_len = nullptr;
        if (metric == L2) O3DML_CUDA(knn_launch<L2, false>(k, KNN_ARGS(out_index, index_is64, out_distance2, no_len)));
        if (metric == L1) O3DML_CUDA(knn_launch<L1, false>(k, KNN_ARGS(out_index, index_is64, out_distance2, no_len)));
        if (metric == LINF) O3DML_CUDA(knn_launch<LINF, false>(k, KNN_ARGS(out_index, index_is64, out_distance2, no_len)));
        return O3DML_OK;
    }
    if (metric == L2) O3DML_CUDA(knn_launch<L2, true>(k, KNN_ARGS((void*)g.idx, 0, g.dist, g.len)));
    if (metric == L1) O3DML_CUDA(knn_launch<L1, true>(k, KNN_ARGS((void*)g.idx, 0, g.dist, g.len)));
    if (metric == LINF) O3DML_CUDA(knn_launch<LINF, true>(k, KNN_ARGS((void*)g.idx, 0, g.dist, g.len)));
#undef KNN_ARGS
    O3DML_CUDA(exclusive_scan_u32(g.len, g.start, num_queries, g.total, g.len_scan_tmp, st));
    O3DML_CUDA(launch<widen_splits_kernel>((unsigned)ceil_div<int64_t>(num_queries, 256), 256, 0, st, g.start,
                                           num_queries, g.total, out_row_splits, d_total));
    O3DML_CUDA(launch<knn_compact_kernel>((unsigned)ceil_div<int64_t>(num_queries * k, 256), 256, 0, st, g.idx, g.dist,
                                          num_queries, k, g.len, g.start, out_index, index_is64, out_distance2));
    return O3DML_OK;
}

// Phase 1 of every radius search: builds the grid (kept in the workspace for phase 2) and writes
// neighbors_row_splits int64 [Nq+1] plus the total (device int64).
static int radius_count_impl(const char* name, const float* points, int64_t num_points,
                             const int64_t* points_row_splits, const float* queries, int64_t num_queries,
                             const int64_t* queries_row_splits, int64_t batch, float radius, const float* radii,
                             int metric, int ignore, int64_t* neighbors_row_splits, int64_t* d_total, void* workspace,
                             size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(radii || radius > 0.f, "%s: radius must be positive", name);
    O3DML_CHECK(batch >= 1 && num_points >= 0 && num_queries >= 0, "%s: bad sizes", name);
    O3DML_CHECK(num_points < ((int64_t)1 << 30), "%s: too many points", name);
    O3DML_CHECK(metric == L2 || metric == L1 || metric == LINF, "%s: unknown metric %d", name, metric);
    Workspace ws(workspace, workspace_bytes);
    const RadiusBuf g = radius_carve(ws, num_points, num_queries, batch);
    if (!ws.ok) O3DML_FAIL(O3DML_ERR_WORKSPACE, "%s: workspace too small (%zu needed)", name, ws.off);
    if (num_queries == 0) {
        O3DML_CUDA(cudaMemsetAsync(neighbors_row_splits, 0, sizeof(int64_t), st));
        if (d_total) O3DML_CUDA(cudaMemsetAsync(d_total, 0, sizeof(int64_t), st));
        return O3DML_OK;
    }
    if (radii) {
        O3DML_CUDA(cudaMemsetAsync(g.item_radius, 0, batch * sizeof(unsigned), st));
        O3DML_CUDA(launch<item_radius_kernel>((unsigned)ceil_div<int64_t>(num_queries, 256), 256, 0, st, radii,
                                              num_queries, queries_row_splits, (int)batch, g.item_radius));
    }
    int rc = grid_build(points, num_points, points_row_splits, queries, num_queries, queries_row_splits, (int)batch,
                        radius, 0, radii ? g.item_radius : nullptr, g, st);
    if (rc) return rc;
    const unsigned nb = (unsigned)ceil_div<int64_t>(num_queries, 128);
    const bool general = radii || metric != L2 || ignore;
    O3DML_CUDA(radius_launch<0>(general, metric, ignore, nb, st, queries, num_queries, queries_row_splits, (int)batch,
                                g.order, g.info, g.cell_start, g.sorted, radius, g.counts, nullptr, nullptr, nullptr,
                                radii, nullptr, 0));
    O3DML_CUDA(exclusive_scan_u32(g.counts, g.counts, num_queries, g.total, g.count_scan_tmp, st));
    O3DML_CUDA(launch<widen_splits_kernel>((unsigned)ceil_div<int64_t>(num_queries, 256), 256, 0, st, g.counts,
                                           num_queries, g.total, neighbors_row_splits, d_total));
    return O3DML_OK;
}

// Phase 2: same workspace (untouched since phase 1), fills the rows.
static int radius_fill_impl(const char* name, const float* queries, int64_t num_points, int64_t num_queries,
                            const int64_t* queries_row_splits, int64_t batch, float radius, const float* radii,
                            int metric, int ignore, int normalize, const int64_t* neighbors_row_splits,
                            void* neighbors_index, int index_is64, float* neighbors_distance, void* workspace,
                            size_t workspace_bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    O3DML_CHECK(metric == L2 || metric == L1 || metric == LINF, "%s: unknown metric %d", name, metric);
    if (num_queries == 0) return O3DML_OK;
    Workspace ws(workspace, workspace_bytes);
    const RadiusBuf g = radius_carve(ws, num_points, num_queries, batch);
    if (!ws.ok) O3DML_FAIL(O3DML_ERR_WORKSPACE, "%s: workspace too small (%zu needed)", name, ws.off);
    O3DML_CHECK(neighbors_index != nullptr && neighbors_distance != nullptr,
                "%s: index and distance outputs are both required", name);
    const unsigned nb = (unsigned)ceil_div<int64_t>(num_queries, 128);
    const bool general = radii || metric != L2 || ignore || normalize || index_is64;
    O3DML_CUDA(radius_launch<1>(general, metric, ignore, nb, st, queries, num_queries, queries_row_splits, (int)batch,
                                g.order, g.info, g.cell_start, g.sorted, radius, nullptr, neighbors_row_splits,
                                index_is64 ? nullptr : (int32_t*)neighbors_index, neighbors_distance, radii,
                                index_is64 ? (int64_t*)neighbors_index : nullptr, normalize));
    return O3DML_OK;
}

}  // namespace o3dml

using namespace o3dml;

extern "C" size_t o3dml_knn_workspace_bytes(int64_t num_points, int64_t num_queries, int64_t batch) {
    return Workspace::measure(knn_carve, num_points, num_queries, batch, 1, 0);
}

extern "C" int o3dml_knn_search(const float* points, int64_t num_points,
                                const int64_t* points_row_splits, const float* queries,
                                int64_t num_queries, const int64_t* queries_row_splits,
                                int64_t batch, int k, void* out_index, int index_is64,
                                float* out_distance2, void* workspace, size_t workspace_bytes,
                                void* stream) {
    return knn_impl("knn_search", points, num_points, points_row_splits, queries, num_queries, queries_row_splits,
                    batch, k, L2, 0, out_index, index_is64, out_distance2, nullptr, nullptr, workspace,
                    workspace_bytes, stream);
}

extern "C" size_t o3dml_knn_search_metric_workspace_bytes(int64_t num_points, int64_t num_queries, int64_t batch,
                                                          int k, int ignore_query_point) {
    return Workspace::measure(knn_carve, num_points, num_queries, batch, k, ignore_query_point ? 1 : 0);
}

extern "C" int o3dml_knn_search_metric(const float* points, int64_t num_points, const int64_t* points_row_splits,
                                       const float* queries, int64_t num_queries, const int64_t* queries_row_splits,
                                       int64_t batch, int k, int metric, int ignore_query_point, void* out_index,
                                       int index_is64, float* out_distance, int64_t* out_row_splits, int64_t* d_total,
                                       void* workspace, size_t workspace_bytes, void* stream) {
    O3DML_CHECK(!ignore_query_point || out_row_splits, "knn_search: ignore_query_point needs out_row_splits");
    return knn_impl("knn_search", points, num_points, points_row_splits, queries, num_queries, queries_row_splits,
                    batch, k, metric, ignore_query_point ? 1 : 0, out_index, index_is64, out_distance, out_row_splits,
                    d_total, workspace, workspace_bytes, stream);
}

extern "C" size_t o3dml_radius_workspace_bytes(int64_t num_points, int64_t num_queries,
                                               int64_t batch) {
    return Workspace::measure(radius_carve, num_points, num_queries, batch);
}

extern "C" int o3dml_radius_count(const float* points, int64_t num_points,
                                  const int64_t* points_row_splits, const float* queries,
                                  int64_t num_queries, const int64_t* queries_row_splits,
                                  int64_t batch, float radius, int64_t* neighbors_row_splits,
                                  int64_t* d_total, void* workspace, size_t workspace_bytes,
                                  void* stream) {
    return radius_count_impl("fixed_radius_search", points, num_points, points_row_splits, queries, num_queries,
                             queries_row_splits, batch, radius, nullptr, L2, 0, neighbors_row_splits, d_total,
                             workspace, workspace_bytes, stream);
}

extern "C" int o3dml_radius_fill(const float* queries, int64_t num_points, int64_t num_queries,
                                 const int64_t* queries_row_splits, int64_t batch, float radius,
                                 const int64_t* neighbors_row_splits, int32_t* neighbors_index,
                                 float* neighbors_distance2, void* workspace,
                                 size_t workspace_bytes, void* stream) {
    return radius_fill_impl("fixed_radius_search", queries, num_points, num_queries, queries_row_splits, batch, radius,
                            nullptr, L2, 0, 0, neighbors_row_splits, neighbors_index, 0, neighbors_distance2,
                            workspace, workspace_bytes, stream);
}

extern "C" int o3dml_radius_search_count(const float* points, int64_t num_points, const int64_t* points_row_splits,
                                         const float* queries, int64_t num_queries,
                                         const int64_t* queries_row_splits, int64_t batch, float radius,
                                         const float* radii, int metric, int ignore_query_point,
                                         int64_t* neighbors_row_splits, int64_t* d_total, void* workspace,
                                         size_t workspace_bytes, void* stream) {
    return radius_count_impl(radii ? "radius_search" : "fixed_radius_search", points, num_points, points_row_splits, queries, num_queries,
                             queries_row_splits, batch, radius, radii, metric, ignore_query_point ? 1 : 0,
                             neighbors_row_splits, d_total, workspace, workspace_bytes, stream);
}

extern "C" int o3dml_radius_search_fill(const float* queries, int64_t num_points, int64_t num_queries,
                                        const int64_t* queries_row_splits, int64_t batch, float radius,
                                        const float* radii, int metric, int ignore_query_point,
                                        int normalize_distances, const int64_t* neighbors_row_splits,
                                        void* neighbors_index, int index_is64, float* neighbors_distance,
                                        void* workspace, size_t workspace_bytes, void* stream) {
    return radius_fill_impl(radii ? "radius_search" : "fixed_radius_search", queries, num_points, num_queries, queries_row_splits, batch, radius,
                            radii, metric, ignore_query_point ? 1 : 0, normalize_distances ? 1 : 0,
                            neighbors_row_splits, neighbors_index, index_is64 ? 1 : 0, neighbors_distance, workspace,
                            workspace_bytes, stream);
}
