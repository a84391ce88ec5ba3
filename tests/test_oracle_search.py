"""The general neighbour-search oracle (oracle/search_ref.c oracle_search_* and its numpy / cKDTree twin in
oracle/search.py): the two restatements agree bit for bit over metric x ignore_query_point x scalar / per-query radii x
normalize x batches with empty items; their row sets equal cKDTree's on tie-free inputs; the L2 scalar case equals the
existing oracle_radius / oracle_knn; and a scalar-radius search and its mirror are each other's inversion."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import ops as O, search as S

P_OF = {0: 2, 1: 1, 2: np.inf}


def cloud(seed, splits_p=(0, 300, 300, 700, 800), splits_q=(0, 120, 170, 170, 330)):
    """Points and queries in four batch items (item 1 has no points, item 2 no queries), with coincident duplicates:
    some queries sit on points, and some points repeat."""
    rng = np.random.default_rng(seed)
    n, m = splits_p[-1], splits_q[-1]
    pts = rng.random((n, 3)).astype(np.float32)
    pts[5:15] = pts[0]                                   # duplicates of one point
    q = rng.random((m, 3)).astype(np.float32) * 1.2 - 0.1  # some queries outside the support box
    q[::7] = pts[rng.integers(0, n, len(q[::7]))]         # queries on support points (maybe of another item)
    q[1] = pts[0]
    return pts, q, np.array(splits_p, np.int64), np.array(splits_q, np.int64)


def radii_for(rng, m):
    r = (rng.random(m) * 0.135 + 0.015).astype(np.float32)    # a 10x spread
    r[1], r[4], r[5], r[6], r[7], r[8] = 0, -0.1, np.nan, np.inf, -0.0, -np.inf
    return r


def equal(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("ignore", [False, True])
@pytest.mark.parametrize("per_query", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
def test_radius_c_equals_numpy(metric, ignore, per_query, normalize):
    pts, q, ps, qs = cloud(1)
    rng = np.random.default_rng(2)
    radii = radii_for(rng, len(q)) if per_query else None
    args = (pts, q, 0.1, radii, ps, qs, metric, ignore, normalize)
    c, n = S.c_search_radius(*args), S.np_search_radius(*args)
    assert equal(c, n)
    assert c[1][-1] > 0
    if per_query:
        rs = c[1]
        lens = np.diff(rs)
        assert lens[4] == lens[5] == lens[6] == lens[8] == 0        # negative, NaN, +inf, -inf radii: empty rows
        # query 1 sits on point 0 and its 10 duplicates with r = 0: it keeps exactly them, normalised to 0 / 0 = NaN
        assert lens[1] == (0 if ignore else 11)
        if normalize:
            assert np.isnan(c[2][rs[1]:rs[2]]).all()
            zero_row = np.repeat(radii == 0, lens)                 # r = +0 or -0
            assert not np.isnan(c[2][~zero_row]).any()


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("ignore", [False, True])
@pytest.mark.parametrize("k", [1, 7, 16])
def test_knn_c_equals_numpy(metric, ignore, k):
    pts, q, ps, qs = cloud(3)
    assert equal(S.c_search_knn(pts, q, k, ps, qs, metric, ignore), S.np_search_knn(pts, q, k, ps, qs, metric, ignore))


def test_knn_ignore_gives_short_rows():
    pts, q, ps, qs = cloud(4)
    idx, d, n = S.c_search_knn(pts, q, 12, ps, qs, 0, True)
    assert n[1] == 12 - 0 and (n <= 12).all()
    # query 1 sits on point 0, which has 10 duplicates: they are all skipped
    assert not np.isin(idx[1], np.arange(5, 15)).any() and 0 not in idx[1]
    small = np.array([0, 3], np.int64)
    idx, d, n = S.c_search_knn(pts[:3], np.concatenate([pts[:3], pts[:1]]), 3, small, np.array([0, 4], np.int64), 1,
                               True)
    assert n.tolist() == [2, 2, 2, 2] and (idx[:, 2] == -1).all() and np.isinf(d[:, 2]).all()


def tie_free(seed, n=400, m=150):
    rng = np.random.default_rng(seed)
    return rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_rows_equal_ckdtree(metric):
    pts, q = tie_free(5)
    tree = cKDTree(pts.astype(np.float64))
    radii = np.random.default_rng(6).uniform(0.05, 0.15, len(q)).astype(np.float32)
    idx, rs, _ = S.c_search_radius(pts, q, 0.0, radii, metric=metric)
    ref = tree.query_ball_point(q.astype(np.float64), radii.astype(np.float64), p=P_OF[metric])
    for i in range(len(q)):
        assert set(idx[rs[i]:rs[i + 1]].tolist()) == set(ref[i])
    nidx, _, _ = S.np_search_knn(pts, q, 10, metric=metric)
    cidx, _, _ = S.c_search_knn(pts, q, 10, metric=metric)
    _, kref = tree.query(q.astype(np.float64), k=10, p=P_OF[metric])
    assert np.array_equal(cidx, kref) and np.array_equal(nidx, kref)


def test_l2_scalar_equals_existing_oracle():
    pts, q, ps, qs = cloud(7)
    idx, rs, d = S.c_search_radius(pts, q, 0.1, None, ps, qs, 0)
    ridx, rrs, rd = O.c_radius(pts, q, 0.1, ps, qs)
    assert np.array_equal(idx, ridx) and np.array_equal(rs, rrs) and np.array_equal(d, rd)
    ps2 = np.array([0, 300, 305, 700, 800], np.int64)      # item 1 has fewer than k points: both pad it alike
    kidx, kd, n = S.c_search_knn(pts, q, 9, ps2, qs, 0)
    oidx, od = O.c_knn(pts, q, 9, ps2, qs)
    assert np.array_equal(kidx, oidx) and np.array_equal(kd, od)
    assert (n[120:170] == 5).all() and (n[:120] == 9).all()


def invert(num, idx, rs):
    """Stable inversion of neighbour lists: for each id, the rows that list it, in row order."""
    rows = np.repeat(np.arange(len(rs) - 1), np.diff(rs))
    o = np.argsort(idx, kind="stable")
    return rows[o], np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=num))]).astype(np.int64)


@pytest.mark.parametrize("metric", [0, 1, 2])
@pytest.mark.parametrize("ignore", [False, True])
def test_mirror_search_is_the_inversion(metric, ignore):
    """The rows of search(points=a, queries=b) inverted equal search(points=b, queries=a) as sets per row: the
    distance is symmetric in (q, p) and so is the coincidence test.  ContinuousConvTranspose's adjoint identity rests
    on this."""
    rng = np.random.default_rng(8)
    a, b = rng.random((300, 3)).astype(np.float32), rng.random((200, 3)).astype(np.float32)
    b[::5] = a[:40]
    fidx, frs, _ = S.c_search_radius(a, b, 0.15, metric=metric, ignore=ignore)
    midx, mrs, _ = S.c_search_radius(b, a, 0.15, metric=metric, ignore=ignore)
    inv, irs = invert(len(a), fidx, frs)
    assert np.array_equal(irs, mrs)
    for i in range(len(a)):
        assert sorted(inv[irs[i]:irs[i + 1]].tolist()) == sorted(midx[mrs[i]:mrs[i + 1]].tolist())
