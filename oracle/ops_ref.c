/*
 * oracle/ops_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, brute-force restatement of the point-cloud operators that the
 * reference (isl-org/Open3D-ML) consumes from the un-vendored `open3d`
 * package.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library.
 *
 * PARITY UNPINNED: the reference tree holds no golden vectors for these ops
 * (SURVEY.md section 8c: tests/test_models.py:73,146,228 assert shapes only) and
 * the upstream implementation (isl-org/Open3D, version not pinned by the
 * reference: ci/run_ci.sh:24 clones `main`) is absent from /root/reference.
 * Semantics therefore follow the reference's CALL SITES
 *   voxelize        ml3d/torch/models/point_pillars.py:328-382
 *   ragged_to_dense ml3d/torch/models/point_pillars.py:364-366, kpconv.py:2030-2032
 *   knn_search      ml3d/datasets/utils/dataprocessing.py:88-103, randlanet.py:218-229
 *   radius search   ml3d/torch/models/kpconv.py:2002-2034
 * plus the published upstream contract (SURVEY.md Appendix C), with the
 * implementation-defined parts fixed as follows (DESIGN.md section "Op contracts"):
 *   - voxelize: a point is kept iff min <= p <= max in every dimension
 *     (inclusive upper bound, which is why point_pillars.py:373-380 must drop
 *     index == extent pillars); coord = (int)((p - min) * (1.0f / voxel_size))
 *     in float32; voxels ordered by ascending linear index
 *     x + ex*(y + ey*z); the first max_voxels survive; inside a voxel point ids
 *     ascend and the first max_points_per_voxel survive.
 *   - neighbour rows (radius and knn) are ordered by (squared distance, index)
 *     ascending; squared distance is float32 ((dx*dx + dy*dy) + dz*dz) with
 *     d = query - point, every operation individually rounded (no FMA);
 *     radius test is d2 <= r*r (float32 product).
 *
 * Build: see oracle/Makefile (gcc -O2 -fopenmp -ffp-contract=off).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))

static inline float sqdist3(const float *q, const float *p) {
    /* volatile stops the compiler from fusing or reassociating */
    volatile float dx = q[0] - p[0];
    volatile float dy = q[1] - p[1];
    volatile float dz = q[2] - p[2];
    volatile float xx = dx * dx;
    volatile float yy = dy * dy;
    volatile float zz = dz * dz;
    volatile float s = xx + yy;
    volatile float t = s + zz;
    return t;
}

/* ---------------------------------------------------------------- knn ---- */
/* Batched exact k-nearest-neighbour search, brute force.
 * points [Np,3], queries [Nq,3], row splits int64 [B+1] each.
 * out_idx [Nq,k] int32 GLOBAL indices into points (-1 pads short batches),
 * out_d2 [Nq,k] float32 (+inf pads).  Order: (d2, idx) ascending. */
EXPORT int oracle_knn(const float *points, const int64_t *p_splits, const float *queries,
                      const int64_t *q_splits, int64_t batch, int k, int32_t *out_idx,
                      float *out_d2) {
    if (k <= 0) return 1;
    for (int64_t b = 0; b < batch; ++b) {
        int64_t p0 = p_splits[b], p1 = p_splits[b + 1];
        int64_t q0 = q_splits[b], q1 = q_splits[b + 1];
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t qi = q0; qi < q1; ++qi) {
            int32_t *bi = out_idx + qi * k;
            float *bd = out_d2 + qi * k;
            int cnt = 0;
            for (int64_t pi = p0; pi < p1; ++pi) {
                float d = sqdist3(queries + 3 * qi, points + 3 * pi);
                if (cnt == k && !(d < bd[k - 1])) continue; /* ties keep the smaller index */
                int j = cnt < k ? cnt : k - 1;
                while (j > 0 && bd[j - 1] > d) { /* strict: equal d keeps earlier index first */
                    bd[j] = bd[j - 1];
                    bi[j] = bi[j - 1];
                    --j;
                }
                bd[j] = d;
                bi[j] = (int32_t)pi;
                if (cnt < k) ++cnt;
            }
            for (int j = cnt; j < k; ++j) {
                bi[j] = -1;
                bd[j] = INFINITY;
            }
        }
    }
    return 0;
}

/* -------------------------------------------------------------- radius ---- */
typedef struct {
    float d;
    int32_t i;
} nb_t;
static int nb_cmp(const void *a, const void *b) {
    const nb_t *x = (const nb_t *)a, *y = (const nb_t *)b;
    if (x->d < y->d) return -1;
    if (x->d > y->d) return 1;
    return (x->i > y->i) - (x->i < y->i);
}

/* Two-phase fixed-radius search.  Phase 1 (out_idx == NULL): fills
 * row_splits int64 [Nq+1].  Phase 2: fills out_idx int32 / out_d2 float32
 * (either may be NULL) following row_splits. */
EXPORT int oracle_radius(const float *points, const int64_t *p_splits, const float *queries,
                         const int64_t *q_splits, int64_t batch, float radius,
                         int64_t *row_splits, int32_t *out_idx, float *out_d2) {
    volatile float r2v = radius * radius;
    const float r2 = r2v;
    int64_t nq = q_splits[batch];
    if (!out_idx && !out_d2) {
        row_splits[0] = 0;
        for (int64_t b = 0; b < batch; ++b) {
            int64_t p0 = p_splits[b], p1 = p_splits[b + 1];
#pragma omp parallel for schedule(dynamic, 64)
            for (int64_t qi = q_splits[b]; qi < q_splits[b + 1]; ++qi) {
                int64_t c = 0;
                for (int64_t pi = p0; pi < p1; ++pi)
                    c += sqdist3(queries + 3 * qi, points + 3 * pi) <= r2;
                row_splits[qi + 1] = c;
            }
        }
        for (int64_t i = 0; i < nq; ++i) row_splits[i + 1] += row_splits[i];
        return 0;
    }
    for (int64_t b = 0; b < batch; ++b) {
        int64_t p0 = p_splits[b], p1 = p_splits[b + 1];
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t qi = q_splits[b]; qi < q_splits[b + 1]; ++qi) {
            int64_t n = row_splits[qi + 1] - row_splits[qi];
            nb_t *tmp = (nb_t *)malloc(sizeof(nb_t) * (size_t)(n > 0 ? n : 1));
            int64_t c = 0;
            for (int64_t pi = p0; pi < p1; ++pi) {
                float d = sqdist3(queries + 3 * qi, points + 3 * pi);
                if (d <= r2 && c < n) {
                    tmp[c].d = d;
                    tmp[c].i = (int32_t)pi;
                    ++c;
                }
            }
            qsort(tmp, (size_t)c, sizeof(nb_t), nb_cmp);
            for (int64_t j = 0; j < c; ++j) {
                if (out_idx) out_idx[row_splits[qi] + j] = tmp[j].i;
                if (out_d2) out_d2[row_splits[qi] + j] = tmp[j].d;
            }
            free(tmp);
        }
    }
    return 0;
}

/* ------------------------------------------------------------ voxelize ---- */
typedef struct {
    int64_t h;
    int64_t i;
} hp_t;
static int hp_cmp(const void *a, const void *b) {
    const hp_t *x = (const hp_t *)a, *y = (const hp_t *)b;
    if (x->h != y->h) return x->h < y->h ? -1 : 1;
    return (x->i > y->i) - (x->i < y->i);
}

/* Hard voxelisation of a batch of clouds (3-D points).
 * Outputs must be sized by the caller for the worst case:
 *   voxel_coords int32 [<=N,3] (x,y,z), point_indices int64 [<=N],
 *   voxel_row_splits int64 [<=N+1], batch_splits int64 [B+1].
 * Returns the number of voxels M via *num_voxels, kept points via *num_kept. */
EXPORT int oracle_voxelize(const float *points, const int64_t *row_splits, int64_t batch,
                           const float *voxel_size, const float *range_min,
                           const float *range_max, int64_t max_points_per_voxel,
                           int64_t max_voxels, int32_t *voxel_coords, int64_t *point_indices,
                           int64_t *voxel_row_splits, int64_t *batch_splits,
                           int64_t *num_voxels, int64_t *num_kept) {
    float inv[3];
    int64_t ext[3];
    for (int d = 0; d < 3; ++d) {
        volatile float iv = 1.0f / voxel_size[d];
        inv[d] = iv;
        volatile float span = range_max[d] - range_min[d];
        volatile float cells = span * inv[d];
        ext[d] = (int64_t)ceilf(cells);
        if (ext[d] < 1) ext[d] = 1;
    }
    int64_t M = 0, L = 0;
    voxel_row_splits[0] = 0;
    batch_splits[0] = 0;
    for (int64_t b = 0; b < batch; ++b) {
        int64_t n0 = row_splits[b], n1 = row_splits[b + 1];
        hp_t *hp = (hp_t *)malloc(sizeof(hp_t) * (size_t)(n1 - n0 > 0 ? n1 - n0 : 1));
        int64_t c = 0;
        for (int64_t i = n0; i < n1; ++i) {
            const float *p = points + 3 * i;
            int ok = 1;
            int64_t ijk[3];
            for (int d = 0; d < 3; ++d) {
                if (!(p[d] >= range_min[d] && p[d] <= range_max[d])) ok = 0;
                volatile float rel = p[d] - range_min[d];
                volatile float sc = rel * inv[d];
                ijk[d] = (int64_t)sc;
            }
            if (!ok) continue;
            /* index == ext can occur for p == max; the linear index stays
             * ordered because (ext+1) is used as the stride */
            hp[c].h = ijk[0] + (ext[0] + 1) * (ijk[1] + (ext[1] + 1) * ijk[2]);
            hp[c].i = i;
            ++c;
        }
        qsort(hp, (size_t)c, sizeof(hp_t), hp_cmp);
        int64_t vox_in_batch = 0;
        int64_t j = 0;
        while (j < c && vox_in_batch < max_voxels) {
            int64_t e = j;
            while (e < c && hp[e].h == hp[j].h) ++e;
            int64_t keep = e - j < max_points_per_voxel ? e - j : max_points_per_voxel;
            int64_t h = hp[j].h;
            voxel_coords[3 * M + 0] = (int32_t)(h % (ext[0] + 1));
            voxel_coords[3 * M + 1] = (int32_t)((h / (ext[0] + 1)) % (ext[1] + 1));
            voxel_coords[3 * M + 2] = (int32_t)(h / ((ext[0] + 1) * (ext[1] + 1)));
            for (int64_t t = 0; t < keep; ++t) point_indices[L++] = hp[j + t].i;
            ++M;
            voxel_row_splits[M] = L;
            ++vox_in_batch;
            j = e;
        }
        batch_splits[b + 1] = M;
        free(hp);
    }
    *num_voxels = M;
    *num_kept = L;
    return 0;
}

/* ------------------------------------------------------- grid subsampling ---- */
/* Per-voxel reduction over CSR voxel lists (the second half of open3d.ml.contrib.subsample /
 * subsample_batch, call sites ml3d/datasets/utils/dataprocessing.py:14-49 and
 * ml3d/torch/models/kpconv.py:2037-2164; upstream = KPConv's grid_subsampling.cpp, barycentre
 * method).  PARITY UNPINNED (no golden vectors in the reference).  Contract fixed here:
 *   - voxels come from oracle_voxelize with range_min = the largest float32 <= floor(min(points) / dl) * dl
 *     over ALL batch items (oracle/ops.py subsample_range), range_max = max(points), no caps -> ascending
 *     linear index per batch item;
 *   - barycentre / feature mean = sequential float32 sum in ascending point id, one division;
 *   - max: a NaN input makes the voxel's max NaN;
 *   - label = most frequent label of the voxel, ties -> smallest label.
 * mode: 0 mean, 1 max, 2 first. */
EXPORT int oracle_voxel_reduce(const float *points, int point_stride, const float *features, int F,
                               const int32_t *labels, const int64_t *vrs, const int64_t *pidx,
                               int64_t M, int pos_mode, int feat_mode, float *out_points,
                               float *out_features, int32_t *out_labels) {
    for (int64_t v = 0; v < M; ++v) {
        int64_t s = vrs[v], e = vrs[v + 1];
        for (int c = 0; c < 3 + F; ++c) {
            int is_pos = c < 3;
            int mode = is_pos ? pos_mode : feat_mode;
            volatile float acc = mode == 1 ? -INFINITY : 0.f;
            for (int64_t j = s; j < e; ++j) {
                float x = is_pos ? points[pidx[j] * point_stride + c] : features[pidx[j] * F + (c - 3)];
                if (mode == 0) acc = acc + x;
                else if (mode == 1) acc = (x > acc || x != x) ? x : acc; /* NaN propagates */
                else if (j == s) acc = x;
            }
            if (mode == 0) acc = acc / (float)(e - s);
            if (is_pos) { if (out_points) out_points[v * 3 + c] = acc; }
            else out_features[v * F + (c - 3)] = acc;
        }
        if (labels) {
            int32_t best = 0;
            int64_t best_n = 0;
            for (int64_t i = s; i < e; ++i) {
                int32_t l = labels[pidx[i]];
                int64_t n = 0;
                for (int64_t j = s; j < e; ++j) n += labels[pidx[j]] == l;
                if (n > best_n || (n == best_n && l < best)) { best = l; best_n = n; }
            }
            out_labels[v] = best;
        }
    }
    return 0;
}

/* ------------------------------------------------------ rotated IoU / NMS ---- */
/* Restates the contract of open3d.ml.torch.ops.nms / contrib.iou_bev / iou_3d as consumed at
 * ml3d/torch/utils/objdet_helper.py:316-350 and ml3d/metrics/mAP.py:85-89 (PARITY UNPINNED: upstream
 * Open3D is absent).  Double precision, Sutherland-Hodgman clipping. */
typedef struct { double cx, cy, w, h, c, s; } rbox_t;

static rbox_t rbox_make(double cx, double cy, double w, double h, double r) {
    rbox_t b = {cx, cy, w, h, cos(r), sin(r)};
    return b;
}
static void rbox_corners(const rbox_t *b, double *x, double *y) {
    const double hw = 0.5 * b->w, hh = 0.5 * b->h;
    const double dx[4] = {-hw, hw, hw, -hw}, dy[4] = {-hh, -hh, hh, hh};
    for (int i = 0; i < 4; ++i) {
        x[i] = b->cx + dx[i] * b->c - dy[i] * b->s;
        y[i] = b->cy + dx[i] * b->s + dy[i] * b->c;
    }
}
/* clipped in a frame centred on a; at most min(area a, area b) */
static double rbox_intersection(const rbox_t *a, const rbox_t *b) {
    if (!(a->w > 0) || !(a->h > 0) || !(b->w > 0) || !(b->h > 0)) return 0.0;
    double px[16], py[16], qx[16], qy[16], bx[4], by[4];
    int n = 4;
    rbox_t a0 = *a, b0 = *b;
    a0.cx = 0; a0.cy = 0;
    b0.cx = b->cx - a->cx; b0.cy = b->cy - a->cy;
    rbox_corners(&a0, px, py);
    rbox_corners(&b0, bx, by);
    for (int e = 0; e < 4 && n > 0; ++e) {
        double x0 = bx[e], y0 = by[e], ex = bx[(e + 1) & 3] - x0, ey = by[(e + 1) & 3] - y0;
        int m = 0;
        double sx = px[n - 1], sy = py[n - 1];
        double sd = ex * (sy - y0) - ey * (sx - x0);
        for (int i = 0; i < n; ++i) {
            double tx = px[i], ty = py[i];
            double td = ex * (ty - y0) - ey * (tx - x0);
            if ((sd >= 0) != (td >= 0)) {
                double t = sd / (sd - td);
                qx[m] = sx + t * (tx - sx); qy[m] = sy + t * (ty - sy); ++m;
            }
            if (td >= 0) { qx[m] = tx; qy[m] = ty; ++m; }
            sx = tx; sy = ty; sd = td;
        }
        n = m;
        for (int i = 0; i < n; ++i) { px[i] = qx[i]; py[i] = qy[i]; }
    }
    if (n < 3) return 0.0;
    double area = 0;
    for (int i = 0; i < n; ++i) {
        int j = (i + 1 == n) ? 0 : i + 1;
        area += px[i] * py[j] - px[j] * py[i];
    }
    area = area > 0 ? 0.5 * area : 0.0;
    const double amin = fmin(a->w * a->h, b->w * b->h);
    return area < amin ? area : amin;
}
static double rbox_iou(const rbox_t *a, const rbox_t *b) {
    double inter = rbox_intersection(a, b);
    double uni = a->w * a->h + b->w * b->h - inter;
    return uni > 0 ? inter / uni : 0.0;
}

/* mode 0: [.,5] (x, y, w, h, r); mode 1: [.,7] (x, y, z, w, h, l, ry) */
EXPORT int oracle_iou_matrix(const float *a, int64_t na, const float *b, int64_t nb, int mode, float *out) {
    for (int64_t i = 0; i < na; ++i)
        for (int64_t j = 0; j < nb; ++j) {
            if (mode == 0) {
                const float *p = a + 5 * i, *q = b + 5 * j;
                rbox_t ra = rbox_make(p[0], p[1], p[2], p[3], p[4]), rb = rbox_make(q[0], q[1], q[2], q[3], q[4]);
                out[i * nb + j] = (float)rbox_iou(&ra, &rb);
            } else {
                const float *p = a + 7 * i, *q = b + 7 * j;
                rbox_t ra = rbox_make(p[0], p[2], p[3], p[5], p[6]), rb = rbox_make(q[0], q[2], q[3], q[5], q[6]);
                double inter2 = rbox_intersection(&ra, &rb);
                double ymax = p[1] < q[1] ? p[1] : q[1];
                double ya = (double)p[1] - p[4], yb = (double)q[1] - q[4];
                double ymin = ya > yb ? ya : yb;
                double ih = ymax - ymin > 0 ? ymax - ymin : 0;
                double va = (double)p[3] * p[4] * p[5], vb = (double)q[3] * q[4] * q[5];
                double inter = fmin(inter2 * ih, fmax(fmin(va, vb), 0.0));
                double uni = va + vb - inter;
                out[i * nb + j] = (float)(uni > 0 ? inter / uni : 0.0);
            }
        }
    return 0;
}

/* boxes [N,5] (x0, y0, x1, y1, r); visiting order = descending score, ties lower index first.
 * margin > 0 additionally reports (via *min_gap) how close any decisive IoU came to thr. */
EXPORT int64_t oracle_nms(const float *boxes, const float *scores, int64_t n, float thr, int64_t *keep,
                          double *min_gap) {
    int64_t *order = (int64_t *)malloc(sizeof(int64_t) * (size_t)(n > 0 ? n : 1));
    for (int64_t i = 0; i < n; ++i) order[i] = i;
    for (int64_t i = 1; i < n; ++i) { /* stable insertion sort, descending score */
        int64_t v = order[i], j = i;
        while (j > 0 && scores[order[j - 1]] < scores[v]) { order[j] = order[j - 1]; --j; }
        order[j] = v;
    }
    int64_t kept = 0;
    double gap = 1e30;
    for (int64_t i = 0; i < n; ++i) {
        const float *p = boxes + 5 * order[i];
        rbox_t a = rbox_make(0.5 * ((double)p[0] + p[2]), 0.5 * ((double)p[1] + p[3]), (double)p[2] - p[0],
                             (double)p[3] - p[1], p[4]);
        int dead = 0;
        for (int64_t k = 0; k < kept && !dead; ++k) {
            const float *q = boxes + 5 * keep[k];
            rbox_t b = rbox_make(0.5 * ((double)q[0] + q[2]), 0.5 * ((double)q[1] + q[3]), (double)q[2] - q[0],
                                 (double)q[3] - q[1], q[4]);
            double iou = rbox_iou(&a, &b);
            double g = fabs(iou - (double)thr);
            if (g < gap) gap = g;
            if (iou > thr) dead = 1;
        }
        if (!dead) keep[kept++] = order[i];
    }
    if (min_gap) *min_gap = gap;
    free(order);
    return kept;
}

/* ------------------------------------------------------------ sparse conv ---- */
/* open3d.ml.torch.layers.SparseConv / SparseConvTranspose as consumed at
 * ml3d/torch/models/sparseconvnet.py:344-485 (PARITY UNPINNED).  Brute force over all (output, input) pairs:
 *   cell_a = floor((in_a - out_a) / v + offset_a + ks_a / 2)   (in / out swapped when transpose)
 *   out[o] += kernel[cell]^T f[in]   for every input whose three cells are in range (ALL of them: on the
 *   voxel-unique inputs the model produces this equals the product's one-input-per-cell table);
 *   normalize: divide by the number of contributing inputs; bias added last.  float64 accumulation. */
EXPORT int oracle_sparse_conv(const float *feat, const float *in_pos, int64_t n, const float *out_pos, int64_t m,
                              float v, const float *offset, const int *ks, int transpose, const float *kernel,
                              int cin, int cout, const float *bias, int normalize, float *out) {
    float inv_v = 1.0f / v;
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t o = 0; o < m; ++o) {
        double *acc = (double *)calloc((size_t)cout, sizeof(double));
        int64_t cnt = 0;
        for (int64_t i = 0; i < n; ++i) {
            int cell[3], ok = 1;
            for (int a = 0; a < 3 && ok; ++a) {
                float d = transpose ? (out_pos[3 * o + a] - in_pos[3 * i + a]) : (in_pos[3 * i + a] - out_pos[3 * o + a]);
                volatile float r0 = d * inv_v;
                volatile float r1 = r0 + offset[a];
                volatile float r = r1 + 0.5f * (float)ks[a];
                int c = (int)floorf(r);
                if (c < 0 || c >= ks[a]) ok = 0;
                cell[a] = c;
            }
            if (!ok) continue;
            ++cnt;
            const float *w = kernel + (size_t)((cell[0] * ks[1] + cell[1]) * ks[2] + cell[2]) * cin * cout;
            for (int ci = 0; ci < cin; ++ci) {
                double f = feat[i * cin + ci];
                for (int co = 0; co < cout; ++co) acc[co] += f * (double)w[ci * cout + co];
            }
        }
        for (int co = 0; co < cout; ++co) {
            double x = acc[co];
            if (normalize && cnt > 0) x /= (double)cnt;
            if (bias) x += bias[co];
            out[o * cout + co] = (float)x;
        }
        free(acc);
    }
    return 0;
}

/* out[i] = sum(values[splits[i] : splits[i+1]]), sequential float32 adds (reduce_subarrays_sum, sparseconvnet.py:318) */
EXPORT int oracle_reduce_subarrays_sum(const float *values, const int64_t *splits, int64_t rows, float *out) {
    for (int64_t i = 0; i < rows; ++i) {
        volatile float acc = 0.f;
        for (int64_t j = splits[i]; j < splits[i + 1]; ++j) acc = acc + values[j];
        out[i] = acc;
    }
    return 0;
}

/* --------------------------------------------------------- continuous conv ---- */
/* open3d.ml.torch.ops.continuous_conv (no call site in the reference; PARITY UNPINNED).  Contract: cconv.cu header.
 * mapping 0 identity / 1 ball_to_cube_radial; interp 0 nearest / 1 linear (clamped) / 2 linear_border. */
EXPORT int oracle_continuous_conv(const float *filters, int sx, int sy, int sz, int cin, int cout,
                                  const float *out_pos, int64_t m, const float *extents, int per_point,
                                  const float *offset, const float *inp_pos, const float *feat,
                                  const float *inp_imp, const int64_t *nbr, const float *nbr_imp,
                                  const int64_t *splits, int align_corners, int mapping, int normalize, int interp,
                                  float *out) {
    const int S[3] = {sx, sy, sz};
    for (int64_t o = 0; o < m; ++o) {
        double *acc = (double *)calloc((size_t)cout, sizeof(double));
        double norm = 0;
        double ext = extents[per_point ? o : 0];
        for (int64_t j = splits[o]; j < splits[o + 1]; ++j) {
            int64_t n = nbr[j];
            double imp = (nbr_imp ? nbr_imp[j] : 1.0) * (inp_imp ? inp_imp[n] : 1.0);
            norm += imp;
            double q[3];
            for (int a = 0; a < 3; ++a)
                q[a] = ((double)inp_pos[3 * n + a] - out_pos[3 * o + a]) * (ext > 0 ? 2.0 / ext : 0.0) + offset[a];
            if (mapping == 1) {
                double n2 = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
                double ni = fmax(fabs(q[0]), fmax(fabs(q[1]), fabs(q[2])));
                double s = ni > 0 ? n2 / ni : 0;
                for (int a = 0; a < 3; ++a) q[a] *= s;
            }
            double u[3];
            for (int a = 0; a < 3; ++a)
                u[a] = align_corners ? (q[a] + 1) * 0.5 * (S[a] - 1) : (q[a] + 1) * 0.5 * S[a] - 0.5;
            int ncorner = interp == 0 ? 1 : 8;
            for (int c = 0; c < ncorner; ++c) {
                int ii[3];
                double w = 1;
                int inside = 1;
                for (int a = 0; a < 3; ++a) {
                    /* the cell is clamped in double before it becomes an int: a far neighbour's floor(u) can be past
                     * the int range.  A NaN u fails both comparisons: cell 0, outside the filter (linear_border
                     * weighs it 0, linear keeps its NaN weight). */
                    double cell;
                    if (interp == 0) {
                        cell = floor(u[a] + 0.5);
                    } else {
                        int bit = (c >> a) & 1;
                        double fl = floor(u[a]);
                        cell = fl + bit;
                        w *= bit ? (u[a] - fl) : 1 - (u[a] - fl);
                    }
                    if (cell >= 0 && cell <= S[a] - 1) {
                        ii[a] = (int)cell;
                    } else {
                        inside = 0;
                        ii[a] = cell > 0 ? S[a] - 1 : 0;
                    }
                }
                if (interp == 2 && !inside) w = 0;
                if (w == 0) continue;
                const float *wt = filters + (size_t)((ii[2] * S[1] + ii[1]) * S[0] + ii[0]) * cin * cout;
                for (int ci = 0; ci < cin; ++ci) {
                    double fv = feat[n * cin + ci] * imp * w;
                    for (int co = 0; co < cout; ++co) acc[co] += fv * wt[ci * cout + co];
                }
            }
        }
        for (int co = 0; co < cout; ++co)
            out[o * cout + co] = (float)((normalize && norm != 0) ? acc[co] / norm : acc[co]);
        free(acc);
    }
    return 0;
}
