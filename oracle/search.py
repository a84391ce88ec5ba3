"""oracle/search.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU checker for the general neighbour searches (radius_search, the L1 / Linf metrics, ignore_query_point,
normalize_distances; contract in DESIGN.md section 2), in the two independent forms of oracle/ops.py:

  * ``c_search_*``  : ctypes bindings of oracle/search_ref.c (brute force)
  * ``np_search_*`` : numpy / scipy restatements (cKDTree candidates in the metric's Minkowski p, then the float32
                      test and ordering of the contract)

PARITY UNPINNED, as for oracle/ops.py: the two are pinned against each other and against cKDTree
(tests/test_oracle_search.py).  Only tests/ may import this module.
"""
import ctypes
import os
import subprocess

import numpy as np

from .ops import _f32, _p, _splits, np_sqdist

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "search_ref.c")
_SO = os.path.join(_HERE, "_build", "libsearch_ref.so")
_LIB = None


def build():
    """Compile oracle/search_ref.c (gcc, the flags of oracle/Makefile) -> oracle/_build/libsearch_ref.so."""
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    gcc = next((g for g in ("/usr/bin/gcc", "/bin/gcc") if os.path.exists(g)), "gcc")
    flags = ["-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden"]
    tmp = "%s.tmp.%d" % (_SO, os.getpid())
    env = {k: v for k, v in os.environ.items() if k not in ("CC", "CXX")}
    if subprocess.run([gcc] + flags + ["-fopenmp", "-o", tmp, _SRC, "-lm"], env=env).returncode != 0:
        subprocess.run([gcc] + flags + ["-o", tmp, _SRC, "-lm"], env=env, check=True)      # no libgomp: serial
    os.replace(tmp, _SO)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
            build()
        _LIB = ctypes.CDLL(_SO)
    return _LIB


# ----------------------------------------------------------------------------
# general neighbour search: metric, one radius per query, ignore_query_point, normalised distances
# (contract: search_ref.c)
# ----------------------------------------------------------------------------
METRICS = {"L2": 0, "L1": 1, "Linf": 2}
_P = {0: 2, 1: 1, 2: np.inf}           # the Minkowski p of each metric, for cKDTree


def c_search_radius(points, queries, radius, radii=None, points_row_splits=None, queries_row_splits=None, metric=0,
                    ignore=False, normalize=False):
    """-> (neighbors_index int64 [L], row_splits int64 [Nq+1], distance float32 [L]); radii None: every query takes
    `radius`."""
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    rd = None if radii is None else _f32(np.asarray(radii).reshape(-1))
    rs = np.zeros(len(queries) + 1, np.int64)
    L = lib()
    args = (_p(points, ctypes.c_float), _p(ps, ctypes.c_int64), _p(queries, ctypes.c_float), _p(qs, ctypes.c_int64),
            ctypes.c_int64(len(ps) - 1), ctypes.c_float(radius), None if rd is None else _p(rd, ctypes.c_float),
            ctypes.c_int(metric), ctypes.c_int(int(ignore)), ctypes.c_int(int(normalize)), _p(rs, ctypes.c_int64))
    assert L.oracle_search_radius(*args, None, None) == 0
    idx = np.empty(int(rs[-1]), np.int64)
    d = np.empty(int(rs[-1]), np.float32)
    assert L.oracle_search_radius(*args, _p(idx, ctypes.c_int64), _p(d, ctypes.c_float)) == 0
    return idx, rs, d


def c_search_knn(points, queries, k, points_row_splits=None, queries_row_splits=None, metric=0, ignore=False):
    """-> (idx int64 [Nq,k] (-1 pads), d float32 [Nq,k] (+inf pads), row lengths int64 [Nq])."""
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    idx = np.empty((len(queries), k), np.int64)
    d = np.empty((len(queries), k), np.float32)
    n = np.zeros(len(queries), np.int64)
    assert lib().oracle_search_knn(_p(points, ctypes.c_float), _p(ps, ctypes.c_int64), _p(queries, ctypes.c_float),
                                   _p(qs, ctypes.c_int64), ctypes.c_int64(len(ps) - 1), ctypes.c_int(k),
                                   ctypes.c_int(metric), ctypes.c_int(int(ignore)), _p(idx, ctypes.c_int64),
                                   _p(d, ctypes.c_float), _p(n, ctypes.c_int64)) == 0
    return idx, d, n


def np_dist(q, p, metric):
    """The distance of the contract in float32, each operation rounded once: q [..., 3] against p [..., 3]."""
    if metric == 0:
        return np_sqdist(q, p)
    a = np.abs((q.astype(np.float32) - p.astype(np.float32)).astype(np.float32))
    if metric == 1:
        return ((a[..., 0] + a[..., 1]).astype(np.float32) + a[..., 2]).astype(np.float32)
    return np.maximum(np.maximum(a[..., 0], a[..., 1]), a[..., 2])       # np.maximum propagates NaN


def _finite(P, Q):
    return bool(np.isfinite(P).all() and np.isfinite(Q).all())


def _coincides(q, p):
    return np.all(q[None, :] == p, axis=1)


def np_search_radius(points, queries, radius, radii=None, points_row_splits=None, queries_row_splits=None, metric=0,
                     ignore=False, normalize=False):
    """cKDTree.query_ball_point candidates (Minkowski p of the metric, one radius per query, 1e-5 relative slack), then
    the float32 test and ordering of the contract."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _np_search_radius(points, queries, radius, radii, points_row_splits, queries_row_splits, metric, ignore,
                                 normalize)


def _np_search_radius(points, queries, radius, radii, points_row_splits, queries_row_splits, metric, ignore,
                      normalize):
    from scipy.spatial import cKDTree
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    r_all = np.full(len(queries), np.float32(radius), np.float32) if radii is None else \
        _f32(np.asarray(radii).reshape(-1))
    rows_i, rows_d = [], []
    for b in range(len(ps) - 1):
        P, Q, R = points[ps[b]:ps[b + 1]], queries[qs[b]:qs[b + 1]], r_all[qs[b]:qs[b + 1]]
        valid = (R >= 0) & np.isfinite(R)
        cand = [[] for _ in range(len(Q))]
        if len(P) and valid.any() and not _finite(P, Q):        # cKDTree takes finite coordinates only
            cand = [np.arange(len(P))] * len(Q)
        elif len(P) and valid.any():
            slack = np.where(valid, R.astype(np.float64) * (1 + 1e-5) + 1e-7, 0.0)
            cand = cKDTree(P).query_ball_point(Q.astype(np.float64), slack, p=_P[metric])
        for qi in range(len(Q)):
            c = np.asarray(cand[qi] if valid[qi] else [], np.int64)
            r = R[qi]
            t = np.float32(r * r) if metric == 0 else r
            if ignore and len(c):
                c = c[~_coincides(Q[qi], P[c])]
            dd = np_dist(Q[qi][None, :], P[c], metric) if len(c) else np.zeros(0, np.float32)
            keep = dd <= t
            c, dd = c[keep], dd[keep]
            o = np.lexsort((c, dd))
            rows_i.append(c[o] + ps[b])
            with np.errstate(invalid="ignore", divide="ignore"):
                rows_d.append((dd[o] / t).astype(np.float32) if normalize else dd[o])
    lens = np.array([len(r) for r in rows_i], np.int64)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.concatenate(rows_i).astype(np.int64) if rows_i else np.zeros(0, np.int64)
    d = np.concatenate(rows_d).astype(np.float32) if rows_d else np.zeros(0, np.float32)
    return idx, rs, d


def np_search_knn(points, queries, k, points_row_splits=None, queries_row_splits=None, metric=0, ignore=False,
                  extra=16):
    """cKDTree.query candidates (Minkowski p of the metric) re-ranked in float32 by (d, idx) after dropping the points
    equal to the query under `ignore`; brute force for a row whose candidate set cannot be proven complete."""
    with np.errstate(over="ignore", invalid="ignore"):
        return _np_search_knn(points, queries, k, points_row_splits, queries_row_splits, metric, ignore, extra)


def _np_search_knn(points, queries, k, points_row_splits, queries_row_splits, metric, ignore, extra):
    from scipy.spatial import cKDTree
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    idx = np.full((len(queries), k), -1, np.int64)
    d = np.full((len(queries), k), np.inf, np.float32)
    n = np.zeros(len(queries), np.int64)
    for b in range(len(ps) - 1):
        P, Q = points[ps[b]:ps[b + 1]], queries[qs[b]:qs[b + 1]]
        if len(P) == 0 or len(Q) == 0:
            continue
        kk = int(min(len(P), k + extra)) if _finite(P, Q) else len(P)       # cKDTree takes finite coordinates only
        if kk < len(P):
            _, cand = cKDTree(P).query(Q.astype(np.float64), k=kk, p=_P[metric])
            cand = np.asarray(cand).reshape(len(Q), kk)
        else:
            cand = np.broadcast_to(np.arange(len(P)), (len(Q), kk))
        for qi in range(len(Q)):
            c = cand[qi]
            complete = kk == len(P)
            while True:
                if ignore:
                    c = c[~_coincides(Q[qi], P[c])]
                dd = np_dist(Q[qi][None, :], P[c], metric)
                ok = ~np.isnan(dd)
                c, dd = c[ok], dd[ok]
                o = np.lexsort((c, dd))
                c, dd = c[o], dd[o]
                # complete when every point was a candidate, or when the worst candidate is clearly beyond the k-th
                if complete or (len(dd) > k and dd[-1] > dd[k - 1] * np.float32(1 + 1e-5)):
                    break
                c, complete = np.arange(len(P)), True
            m = min(k, len(c))
            g = qs[b] + qi
            idx[g, :m], d[g, :m], n[g] = c[:m] + ps[b], dd[:m], m
    return idx, d, n
