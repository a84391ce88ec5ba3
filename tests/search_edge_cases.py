"""Neighbour-search cases at the edges of the hash-grid searches of grid.cu (k-NN, fixed-radius and per-query radius
search), shared by tests/test_oracle_search_edges.py (the two oracle restatements and a float64 brute force) and
tests/test_gpu_search_edges.py (the kernels, bit-equal to the oracle).  Every builder is seeded and returns a Case:
points, queries, their int64 row splits, one scalar radius, one radius per query and the k values to search with.

  nonfinite    NaN, +inf and -inf in points and queries inside one batch item; an item of exactly 16 points, one of
               them NaN; a pair of points 1e20 apart, whose float32 L2 distance overflows to +inf
  identical    every point the same
  line         200 000 points on a 100 m line: about 3.3e5 cells on one axis
  plane        points on a plane
  clusters     two clusters 1e4 m apart, with queries between them
  far5e5, far1e7  clouds offset by 5e5 and 1e7, where the float32 ulp is 1/16 m and 1 m: coordinates are quantised, so
               distance ties are common (rows order them by index), and some radii are below the ulp
  outside      queries up to 1e3 x the extent outside the bounding box, in every direction
  kedges       k at each knn_kernel instance edge (1, 2, 8, 9, 16, 17, 32, 33, 64), with items of k and k - 1 points
  batch        120 items mixing empty items, one-point items and items without queries, over more than 4096 cells
               and 4096 queries, so that the scans run over many tiles
  stoprule     the line, with queries whose k-th neighbour sits within 1e-3 cells of a ring boundary of the k-NN walk

Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
from collections import namedtuple

import numpy as np

F32 = np.float32
KEDGES = (1, 2, 8, 9, 16, 17, 32, 33, 64)

Case = namedtuple("Case", "points queries ps qs radius radii ks")


def f32(a):
    return np.ascontiguousarray(a, F32)


def _case(pts, q, ps, qs, radius, rng, ks=(1, 9, 33), spread=(0.3, 3.0), radii=None):
    """A Case whose per-query radii spread over `spread` x radius, with 0, -r, NaN and +inf at queries 1..4."""
    q = f32(q)
    if radii is None:
        radii = f32(rng.uniform(*spread, len(q)) * radius)
        for i, v in zip(range(1, 5), (0.0, -radius, np.nan, np.inf)):
            if i < len(q):
                radii[i] = v
    return Case(f32(pts), q, np.asarray(ps, np.int64), np.asarray(qs, np.int64), float(F32(radius)), f32(radii),
                tuple(ks))


def one(pts, q):
    return [0, len(pts)], [0, len(q)]


# ------------------------------------------------------------------------------------------------- builders
def nonfinite(seed=0):
    rng = np.random.default_rng(seed)
    a = rng.random((1500, 3)).astype(F32)
    bad = rng.choice(1500, 60, replace=False)
    for j, i in enumerate(bad):                             # one non-finite coordinate, or a whole non-finite point
        v = (np.nan, np.inf, -np.inf)[j % 3]
        if j % 4 == 3:
            a[i] = v
        else:
            a[i, j % 3] = v
    qa = rng.random((300, 3)).astype(F32) * 1.2 - 0.1
    qa[::5] = a[rng.integers(0, 1500, len(qa[::5]))]        # on points, some of them non-finite
    for j in range(24):                                     # non-finite queries
        qa[10 + j, j % 3] = (np.nan, np.inf, -np.inf)[j % 3]
    qa[40:43] = [np.nan, np.inf, -np.inf]
    b = rng.random((16, 3)).astype(F32)                     # exactly 16 points, one of them NaN
    b[7, 1] = np.nan
    qb = np.concatenate([rng.random((40, 3)), b[:5]]).astype(F32)
    c = rng.random((200, 3)).astype(F32)                    # a pair 1e20 apart: L2 overflows, L1 / Linf do not
    c[0] = [1e20, 0, 0]
    c[1] = [-1e20, 0.5, 0.5]
    c[2] = [0, 3e19, 0]
    qc = np.concatenate([rng.random((40, 3)), c[:3], [[1e20, 1e20, 1e20]]]).astype(F32)
    pts = np.concatenate([a, b, c])
    q = np.concatenate([qa, qb, qc])
    ps = [0, 1500, 1516, 1716]
    qs = [0, len(qa), len(qa) + len(qb), len(q)]
    c = _case(pts, q, ps, qs, 0.15, rng, ks=(1, 9, 16, 17, 64))
    c.radii[qs[2]:qs[2] + 20] = 3e38                        # r * r = +inf: every distance but NaN is within
    return c


def identical(seed=1):
    rng = np.random.default_rng(seed)
    p = np.full((3000, 3), [1.25, -3.5, 7.0], F32)
    q = np.concatenate([p[:50], p[0] + rng.normal(0, 0.1, (100, 3)), p[0] + rng.normal(0, 100, (50, 3))])
    return _case(p, q, *one(p, q), 0.1, rng, ks=(1, 9, 64))


LINE_N = 200_000


def line_points(seed):
    rng = np.random.default_rng(seed)
    p = np.zeros((LINE_N, 3), F32)
    p[:, 0] = rng.uniform(0, 100, LINE_N)
    p[:, 1], p[:, 2] = 0.5, -0.25
    return p


def line(seed=2):
    rng = np.random.default_rng(seed)
    p = line_points(seed)
    q = np.concatenate([p[rng.integers(0, LINE_N, 60)],
                        np.stack([rng.uniform(-1, 101, 100), np.full(100, 0.5), np.full(100, -0.25)], 1),
                        rng.uniform(-1, 101, (40, 3))]).astype(F32)
    return _case(p, q, *one(p, q), 0.002, rng, ks=(1, 16, 64))


def plane(seed=3):
    rng = np.random.default_rng(seed)
    p = np.zeros((8000, 3), F32)
    p[:, :2] = rng.uniform(0, 10, (8000, 2))
    p[:, 2] = 1.5
    q = np.concatenate([p[rng.integers(0, 8000, 100)], rng.uniform(-1, 11, (200, 3))]).astype(F32)
    q[100:200, 2] = 1.5
    return _case(p, q, *one(p, q), 0.1, rng)


def clusters(seed=4):
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 1, (2000, 3))
    b = rng.normal(0, 1, (2000, 3)) + [1e4, 0, 0]
    p = np.concatenate([a, b]).astype(F32)
    t = rng.random(150)[:, None]
    q = np.concatenate([t * [1e4, 0, 0] + rng.normal(0, 1, (150, 3)), p[rng.integers(0, 4000, 100)]])
    q[:3] = [[5e3, 0, 0], [5e3 + 1, 0, 0], [5e3 - 1, 0, 0]]     # about the middle: a near tie between the clusters
    return _case(p, q, *one(p, q), 0.3, rng, spread=(0.3, 3e4))


def far(offset, seed):
    rng = np.random.default_rng(seed)
    ulp = float(np.spacing(F32(offset)))
    p = (rng.uniform(0, 40 * ulp, (3000, 3)) + offset).astype(F32)     # about 40 distinct values per axis
    p[100:110] = p[0]
    q = np.concatenate([p[rng.integers(0, 3000, 200)],
                        rng.uniform(-4 * ulp, 44 * ulp, (200, 3)) + offset]).astype(F32)
    radii = f32(rng.choice([0.25, 0.5, 1.0, 2.0, 4.0], len(q)) * ulp)  # some below the ulp
    radii[1:5] = [0.0, -ulp, np.nan, np.inf]
    return _case(p, q, *one(p, q), 3 * ulp, rng, radii=radii)


def far5e5(seed=5):
    return far(5e5, seed)


def far1e7(seed=6):
    return far(1e7, seed)


def outside(seed=7):
    rng = np.random.default_rng(seed)
    p = rng.random((3000, 3)).astype(F32) * [2.0, 1.0, 0.5] - [1.0, 0.5, 0.0]
    lo, hi = p.min(0), p.max(0)
    c, ext = (lo + hi) / 2, hi - lo
    dirs = np.array([[i, j, k] for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)])
    q = [c + d * s * ext for d in dirs for s in (0.51, 0.6, 2.0, 10.0, 100.0, 1000.0)]
    q = np.concatenate([np.array(q), c + rng.normal(0, 1, (200, 3)) * ext * 10.0 ** rng.integers(0, 4, (200, 1))])
    return _case(p, q, *one(p, q), 0.2, rng, spread=(0.3, 3e3))


def kedges(seed=8):
    rng = np.random.default_rng(seed)
    sizes = [n for k in KEDGES for n in (k, k - 1)] + [1200]
    pts = [rng.random((n, 3)) for n in sizes]
    qs_ = [np.concatenate([rng.random((20, 3)), x[:3]]) for x in pts]
    ps = np.concatenate([[0], np.cumsum(sizes)])
    qs = np.concatenate([[0], np.cumsum([len(x) for x in qs_])])
    return _case(np.concatenate(pts), np.concatenate(qs_), ps, qs, 0.2, rng, ks=KEDGES)


def batch(seed=9):
    rng = np.random.default_rng(seed)
    nb = 120
    npts = rng.integers(50, 400, nb)
    npts[::7], npts[3::11] = 0, 1                           # empty items, one-point items
    nq = rng.integers(30, 90, nb)
    nq[5::9] = 0                                            # items without queries
    pts, q = [], []
    for b in range(nb):
        o = rng.uniform(-50, 50, 3)
        pts.append(rng.random((npts[b], 3)) * rng.uniform(0.5, 4) + o)
        qq = rng.random((nq[b], 3)) * 4 + o - 1
        if npts[b] and nq[b]:
            qq[::4] = pts[b][rng.integers(0, npts[b], len(qq[::4]))]
        q.append(qq)
    ps = np.concatenate([[0], np.cumsum(npts)])
    qs = np.concatenate([[0], np.cumsum(nq)])
    return _case(np.concatenate(pts), np.concatenate(q), ps, qs, 0.3, rng, ks=(1, 8, 33))


# ------------------------------------------------------------------------ cell size of the k-NN grid (host replica)
def knn_cell_size(points, k):
    """grid_setup_kernel's k-NN cell size and grid dims for one batch item, in its float32 / float64 arithmetic:
    the radius expected to hold max(k, 4) points at the bounding box's surface or volume density, at least 1e-6 and
    2^-20 of the longest side, grown by 1.26 until the cells fit 2 n + 64."""
    p = f32(points)
    n = len(p)
    e = np.maximum((p.max(0) - p.min(0)).astype(F32), F32(1e-6))
    e0, e2 = e.max(), e.min()
    e1 = F32(F32(F32(F32(e[0] + e[1]) + e[2]) - e0) - e2)
    kk = F32(max(k, 4))
    with np.errstate(invalid="ignore"):     # e1 rounds below 0 on a line: NaN, which fmaxf drops
        cs2 = np.sqrt(F32(F32(F32(kk * e0) * e1) / F32(F32(3.14159265) * F32(n))))
    cs3 = np.cbrt(F32(F32(F32(F32(kk * e0) * e1) * e2) / F32(F32(4.18879) * F32(n))))
    cs = np.fmax(np.fmax(cs2, cs3), F32(1e-6))
    cs = np.fmax(cs, F32(e0 * F32(2.0 ** -20)))
    cap = 2.0 * n + 64.0
    for _ in range(64):
        if np.prod(np.floor(e.astype(np.float64) / float(cs)) + 1) <= cap:
            break
        cs = F32(cs * F32(1.26))
    dims = (np.floor(e.astype(np.float64) / float(cs)) + 1).astype(np.int64)
    return F32(cs), dims


STOP_K = 16


def stoprule(seed=10, k=STOP_K, want=200, tol=1e-3):
    """Queries on the line whose k-th neighbour (in |dx|, the distance of every metric on the line) lies within `tol`
    cells of r * cs or of the walk's stop bound 0.9999 r * cs, for some ring r >= 1."""
    rng = np.random.default_rng(seed)
    p = line_points(seed)
    cs, _ = knn_cell_size(p, k)
    xs = np.sort(p[:, 0].astype(np.float64))
    cand = f32(rng.uniform(0, 100, 400_000)).astype(np.float64)
    pos = np.searchsorted(xs, cand)
    win = np.clip(pos[:, None] + np.arange(-k, k)[None, :], 0, LINE_N - 1)
    dk = np.sort(np.abs(xs[win] - cand[:, None]), axis=1)[:, k - 1]
    hit = np.zeros(len(cand), bool)
    for scale in (1.0, 0.9999):
        t = dk / (float(cs) * scale)
        hit |= (np.abs(t - np.round(t)) < tol) & (np.round(t) >= 1)
    x = cand[hit][:want]
    q = np.stack([x, np.full(len(x), 0.5), np.full(len(x), -0.25)], 1)
    return _case(p, q, *one(p, q), 0.002, rng, ks=(k,))


BUILDERS = {f.__name__: f for f in (nonfinite, identical, line, plane, clusters, far5e5, far1e7, outside, kedges, batch,
                                    stoprule)}
FINITE = ("identical", "line", "plane", "clusters", "far5e5", "far1e7", "outside", "kedges", "batch", "stoprule")

_CACHE = {}


def case(name):
    """The builder's Case, built once per process."""
    if name not in _CACHE:
        _CACHE[name] = BUILDERS[name]()
    return _CACHE[name]


def short_items(c, k):
    """True when some batch item holds fewer than k points (knn_search then needs allow_short)."""
    return bool((np.diff(c.ps) < k).any())
