/*
 * oracle/search_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, brute-force restatement of the general neighbour searches (radius_search / fixed_radius_search /
 * knn_search with a metric, one radius per query, ignore_query_point and normalised distances), the companion of
 * oracle/ops_ref.c, whose L2 fixed-radius and k-NN oracles it extends.  Only tests/ may load this library.
 * PARITY UNPINNED (see the header of ops_ref.c); the contract is written down in DESIGN.md section 2.
 *
 * Build: oracle/search.py (gcc -O2 -fopenmp -ffp-contract=off, as oracle/Makefile builds ops_ref.c).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#define EXPORT __attribute__((visibility("default")))

/* the squared distance and row order of ops_ref.c (sqdist3, nb_cmp) */
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

/* ------------------------------------------------- general neighbour search ---- */
/* radius_search / fixed_radius_search / knn_search with a metric, one radius per query and
 * ignore_query_point (DESIGN.md section 2, PARITY UNPINNED).  d = q - p per axis, each difference
 * rounded once, no FMA:
 *   metric 0 (L2)   ((dx*dx + dy*dy) + dz*dz), squared;
 *   metric 1 (L1)   (|dx| + |dy|) + |dz|;
 *   metric 2 (Linf) max(max(|dx|, |dy|), |dz|), NaN when a difference is NaN.
 * Radius: kept when d <= t, t = r*r (rounded once) for L2 and r otherwise; radii (may be NULL: every
 * query takes `radius`) with a negative, NaN or infinite entry give an empty row; normalize returns
 * d / t (L2) or d / r.  ignore: skip every point whose three coordinates equal the query's.
 * Rows ascend by (d, index); a NaN d is never kept nor ranked. */
static inline float maxnan(float a, float b) { return (a != a || b != b) ? NAN : (a > b ? a : b); }

static inline float metric_dist(const float *q, const float *p, int metric) {
    if (metric == 0) return sqdist3(q, p);
    volatile float dx = q[0] - p[0];
    volatile float dy = q[1] - p[1];
    volatile float dz = q[2] - p[2];
    float ax = fabsf(dx), ay = fabsf(dy), az = fabsf(dz);
    if (metric == 1) {
        volatile float s = ax + ay;
        volatile float t = s + az;
        return t;
    }
    return maxnan(maxnan(ax, ay), az);
}

static inline int coincides(const float *q, const float *p) { return q[0] == p[0] && q[1] == p[1] && q[2] == p[2]; }

/* Phase 1 (out_idx == NULL): row_splits int64 [Nq+1].  Phase 2: out_idx int64 [L], out_d float32 [L]. */
EXPORT int oracle_search_radius(const float *points, const int64_t *p_splits, const float *queries,
                                const int64_t *q_splits, int64_t batch, float radius, const float *radii,
                                int metric, int ignore, int normalize, int64_t *row_splits, int64_t *out_idx,
                                float *out_d) {
    int64_t nq = q_splits[batch];
    if (!out_idx) row_splits[0] = 0;
    for (int64_t b = 0; b < batch; ++b) {
        int64_t p0 = p_splits[b], p1 = p_splits[b + 1];
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t qi = q_splits[b]; qi < q_splits[b + 1]; ++qi) {
            const float r = radii ? radii[qi] : radius;
            const int valid = r >= 0.f && r <= 3.402823466e38f;
            volatile float rr = r * r;
            const float t = metric == 0 ? rr : r;
            const float *q = queries + 3 * qi;
            nb_t *tmp = out_idx ? (nb_t *)malloc(sizeof(nb_t) * (size_t)(p1 - p0 > 0 ? p1 - p0 : 1)) : NULL;
            int64_t c = 0;
            for (int64_t pi = p0; valid && pi < p1; ++pi) {
                if (ignore && coincides(q, points + 3 * pi)) continue;
                float d = metric_dist(q, points + 3 * pi, metric);
                if (d <= t) {
                    if (tmp) { tmp[c].d = d; tmp[c].i = (int32_t)pi; }
                    ++c;
                }
            }
            if (!tmp) {
                row_splits[qi + 1] = c;
                continue;
            }
            qsort(tmp, (size_t)c, sizeof(nb_t), nb_cmp);
            for (int64_t j = 0; j < c; ++j) {
                volatile float dn = tmp[j].d / t;
                out_idx[row_splits[qi] + j] = tmp[j].i;
                out_d[row_splits[qi] + j] = normalize ? dn : tmp[j].d;
            }
            free(tmp);
        }
    }
    if (!out_idx)
        for (int64_t i = 0; i < nq; ++i) row_splits[i + 1] += row_splits[i];
    return 0;
}

/* k nearest: out_idx int64 [Nq,k] (-1 pads), out_d float32 [Nq,k] (+inf pads), out_len int64 [Nq] = the
 * neighbours found (fewer than k when the item is smaller, ignore skipped points or distances were NaN).  A NaN d is
 * never ranked; +inf ranks after every finite d.  The k best are kept in a sorted buffer: a point enters when it sorts
 * before the buffer's last entry (or the buffer is not full), the order of a full sort by (d, index). */
EXPORT int oracle_search_knn(const float *points, const int64_t *p_splits, const float *queries,
                             const int64_t *q_splits, int64_t batch, int k, int metric, int ignore,
                             int64_t *out_idx, float *out_d, int64_t *out_len) {
    if (k <= 0) return 1;
    for (int64_t b = 0; b < batch; ++b) {
        int64_t p0 = p_splits[b], p1 = p_splits[b + 1];
#pragma omp parallel for schedule(dynamic, 64)
        for (int64_t qi = q_splits[b]; qi < q_splits[b + 1]; ++qi) {
            const float *q = queries + 3 * qi;
            nb_t *best = (nb_t *)malloc(sizeof(nb_t) * (size_t)k);
            int64_t n = 0;
            for (int64_t pi = p0; pi < p1; ++pi) {
                if (ignore && coincides(q, points + 3 * pi)) continue;
                nb_t c = {metric_dist(q, points + 3 * pi, metric), (int32_t)pi};
                if (c.d != c.d) continue;
                if (n == k && nb_cmp(&c, &best[k - 1]) >= 0) continue;
                int64_t j = n < k ? n++ : k - 1;
                while (j > 0 && nb_cmp(&c, &best[j - 1]) < 0) {
                    best[j] = best[j - 1];
                    --j;
                }
                best[j] = c;
            }
            for (int64_t j = 0; j < k; ++j) {
                out_idx[qi * k + j] = j < n ? best[j].i : -1;
                out_d[qi * k + j] = j < n ? best[j].d : INFINITY;
            }
            out_len[qi] = n;
            free(best);
        }
    }
    return 0;
}
