"""The neighbour-search oracle at the edges of tests/search_edge_cases.py: the C brute force (oracle/search_ref.c) and
the numpy / cKDTree restatement (oracle/search.py) agree bit for bit on every builder, metric and ignore_query_point;
on every finite builder, each k-NN and radius row holds the points a float64 brute force puts there, up to float32
rounding of the distance; the non-finite rule (NaN never ranked nor within a radius, +inf ranked after every finite
distance, rows short and -1 / +inf padded) holds; and the host replica of the k-NN cell size reaches the grid sizes
the line case is built for."""
import numpy as np
import pytest

import search_edge_cases as E
from oracle import search as S

METRICS = [0, 1, 2]
TOL = 16 * 2.0 ** -24    # float32 distance vs float64: a few roundings of relative size 2^-24 each


def equal(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


@pytest.mark.parametrize("name", list(E.BUILDERS))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_knn_c_equals_numpy(name, metric, ignore):
    c = E.case(name)
    for k in c.ks:
        a = S.c_search_knn(c.points, c.queries, k, c.ps, c.qs, metric, ignore)
        b = S.np_search_knn(c.points, c.queries, k, c.ps, c.qs, metric, ignore)
        assert equal(a, b), k


@pytest.mark.parametrize("name", list(E.BUILDERS))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_radius_c_equals_numpy(name, metric, ignore):
    c = E.case(name)
    for radius, radii, normalize in ((c.radius, None, False), (0.0, c.radii, ignore)):
        args = (c.points, c.queries, radius, radii, c.ps, c.qs, metric, ignore, normalize)
        assert equal(S.c_search_radius(*args), S.np_search_radius(*args))


def dist64(q, p, metric):
    """Distances of the float32 coordinates in float64 (L2 squared, as the searches return it)."""
    d = np.abs(q[None, :].astype(np.float64) - p.astype(np.float64))
    return (d * d).sum(1) if metric == 0 else d.sum(1) if metric == 1 else d.max(1)


def rows(c):
    """(query, item's first point, item's points) of every query."""
    for b in range(len(c.ps) - 1):
        P = c.points[c.ps[b]:c.ps[b + 1]]
        for qi in range(c.qs[b], c.qs[b + 1]):
            yield qi, c.ps[b], P


@pytest.mark.parametrize("name", E.FINITE)
@pytest.mark.parametrize("metric", METRICS)
def test_rows_hold_the_float64_nearest(name, metric):
    """Every point a float64 brute force puts clearly inside a row is in it, and nothing clearly outside is: the
    float32 contract hides no wrong neighbour at large offsets, sizes or distances.  Ties and near-ties (within the
    float32 rounding of the distance) may go either way."""
    c = E.case(name)
    k = max(c.ks)
    idx, _, n = S.c_search_knn(c.points, c.queries, k, c.ps, c.qs, metric)
    ridx, rs, _ = S.c_search_radius(c.points, c.queries, 0.0, c.radii, c.ps, c.qs, metric)
    for qi, p0, P in rows(c):
        if not len(P):
            assert n[qi] == 0 and rs[qi + 1] == rs[qi]
            continue
        d = dist64(c.queries[qi], P, metric)
        m = min(k, len(P))
        assert n[qi] == m
        got = idx[qi, :m] - p0
        kth = np.partition(d, m - 1)[m - 1]
        assert (d[got] <= kth * (1 + TOL)).all(), qi
        assert np.isin(np.flatnonzero(d < kth * (1 - TOL)), got).all(), qi
        r = np.float64(c.radii[qi])
        if not (r >= 0 and np.isfinite(r)):
            assert rs[qi + 1] == rs[qi]
            continue
        t = r * r if metric == 0 else r
        got = ridx[rs[qi]:rs[qi + 1]] - p0
        assert (d[got] <= t * (1 + TOL)).all(), qi
        assert np.isin(np.flatnonzero(d < t * (1 - TOL)), got).all(), qi


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_nonfinite_rule(metric, ignore):
    """NaN distances are never ranked nor within a radius; +inf ranks after every finite distance; rows run short."""
    c = E.case("nonfinite")
    k = 16
    idx, d, n = S.c_search_knn(c.points, c.queries, k, c.ps, c.qs, metric, ignore)
    assert ((idx >= -1) & (idx < len(c.points))).all()
    assert not np.isnan(d).any()
    for qi, p0, P in rows(c):
        with np.errstate(over="ignore", invalid="ignore"):
            dd = S.np_dist(c.queries[qi][None, :], P, metric)
        keep = ~np.isnan(dd)
        if ignore:
            keep &= ~np.all(P == c.queries[qi], axis=1)
        m = min(k, int(keep.sum()))
        assert n[qi] == m
        assert (idx[qi, m:] == -1).all() and np.isposinf(d[qi, m:]).all()
        assert not np.isnan(dd[idx[qi, :m] - p0]).any()
        # a +inf distance comes after every finite one
        fin = np.isfinite(dd) & keep
        assert (np.isfinite(d[qi, :m]) == (np.arange(m) < min(m, int(fin.sum())))).all()
    # the item of 16 points with one NaN: every row there holds 15 neighbours (fewer when ignore skips the query)
    item = np.arange(c.qs[1], c.qs[2])
    assert (n[item] <= 15).all() and (n[item[:40]] == 15).all() and (idx[item, 15] == -1).all()
    # L2 between points 1e20 apart overflows to +inf: ranked, after every finite distance (L1 / Linf stay finite)
    q = c.qs[2] + 40                                        # the query on (1e20, 0, 0)
    assert n[q] == k and (idx[q] >= c.ps[2]).all()
    assert np.isposinf(d[q, 0 if ignore else 1:]).all() == (metric == 0)
    # a radius of 3e38: t = r * r = +inf for L2, so +inf distances are within it; every non-NaN distance is, anyway
    ridx, rs, rd = S.c_search_radius(c.points, c.queries, 0.0, c.radii, c.ps, c.qs, metric, ignore)
    for qi in range(c.qs[2], c.qs[2] + 20):
        assert rs[qi + 1] - rs[qi] == 200 - (ignore and (c.points[c.ps[2]:] == c.queries[qi]).all(1).any())
    assert np.isposinf(rd[rs[c.qs[2]]:rs[c.qs[2] + 20]]).any() == (metric == 0)


def test_cell_size_replica_reaches_the_line_grid():
    """The line has about 3.3e5 cells along x; the stop-rule queries sit within 1e-3 cells of a ring boundary."""
    c = E.case("line")
    cs, dims = E.knn_cell_size(c.points, E.STOP_K)
    assert dims[0] > 3e5 and (dims[1:] == 1).all() and dims[0] <= 2 * E.LINE_N + 64
    s = E.case("stoprule")
    assert len(s.queries) == 200
    d = np.sort(np.abs(s.points[:, 0].astype(np.float64)[None, :] - s.queries[:20, :1].astype(np.float64)), 1)
    t = d[:, E.STOP_K - 1] / float(cs)
    near = np.minimum(np.abs(t - np.round(t)), np.abs(t / 0.9999 - np.round(t / 0.9999)))
    assert (near < 1.01e-3).all()


def test_batch_runs_the_scans_over_many_tiles():
    c = E.case("batch")
    sizes = np.diff(c.ps)
    assert len(sizes) >= 100 and (sizes == 0).any() and (sizes == 1).any() and (np.diff(c.qs) == 0).any()
    assert 2 * len(c.points) + 64 * len(sizes) > 4096 and len(c.queries) > 4096
