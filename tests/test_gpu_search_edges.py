"""The neighbour searches of grid.cu at the edges of tests/search_edge_cases.py (non-finite coordinates, degenerate and
far-from-origin clouds, queries far outside the box, k at each knn_kernel instance edge, large batches, queries at the
k-NN walk's ring boundaries), bit-equal to the C oracle (oracle/search.py c_search_*): index, row splits and distances
of knn_search (every metric, with and without ignore_query_point, int32 and int64 ids; the plain L2 path is
o3dml_knn_search, RandLA-Net's), fixed_radius_search (its L2 / int32 / one-radius path is the non-GENERAL radius_kernel,
KPFCNN's) and radius_search, and of the search layers.  Indices are range-checked and compared, never gathered with."""
import functools

import numpy as np
import pytest
import torch

import open3d_ml_b200 as M
import search_edge_cases as E
from oracle import search as S

pytestmark = pytest.mark.gpu

METRICS = ["L2", "L1", "Linf"]
INDEX_DTYPES = (torch.int32, torch.int64)


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def device_case(name):
    c = E.case(name)
    return T(c.points), T(c.queries), T(c.ps), T(c.qs), T(c.radii)


@functools.lru_cache(maxsize=None)
def ref_knn(name, k, metric, ignore):
    c = E.case(name)
    return S.c_search_knn(c.points, c.queries, k, c.ps, c.qs, S.METRICS[metric], ignore)


def host_ids(t, n):
    """The ids as int64 on the host, after checking that each is -1 or a row of the n points."""
    a = t.cpu().numpy().astype(np.int64)
    bad = (a < -1) | (a >= n)
    assert not bad.any(), "ids out of range: %s" % np.unique(a[bad])[:8]
    return a


def check_knn(res, ref, k, ignore, n, index_dtype):
    ref_idx, ref_d, ref_n = ref
    assert res.neighbors_index.dtype == index_dtype and res.neighbors_index.is_cuda
    if ignore:
        keep = np.arange(k)[None, :] < ref_n[:, None]
        want_rs, want_idx, want_d = np.concatenate([[0], np.cumsum(ref_n)]), ref_idx[keep], ref_d[keep]
    else:
        want_rs, want_idx, want_d = np.arange(len(ref_n) + 1) * k, ref_idx.reshape(-1), ref_d.reshape(-1)
    got = host_ids(res.neighbors_index, n)
    assert got.shape == want_idx.shape
    wrong = np.flatnonzero(got != want_idx)
    assert not len(wrong), "%d ids differ, first at %d: %d for %d" % (len(wrong), wrong[0], got[wrong[0]],
                                                                       want_idx[wrong[0]])
    assert np.array_equal(res.neighbors_row_splits.cpu().numpy(), want_rs)
    assert np.array_equal(res.neighbors_distance.cpu().numpy(), want_d)


@pytest.mark.parametrize("name", list(E.BUILDERS))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_knn_search_bit_equal_to_oracle(name, metric, ignore):
    c = E.case(name)
    p, q, ps, qs, _ = device_case(name)
    for k in c.ks:
        ref = ref_knn(name, k, metric, ignore)
        for index_dtype in INDEX_DTYPES:
            res = M.ops.knn_search(p, q, k, ps, qs, index_dtype=index_dtype, metric=metric, ignore_query_point=ignore,
                                   return_distances=True, allow_short=E.short_items(c, k))
            check_knn(res, ref, k, ignore, len(c.points), index_dtype)


def check_radius(res, ref, n, index_dtype):
    idx, rs, d = ref
    assert res.neighbors_index.dtype == index_dtype and res.neighbors_index.is_cuda
    assert np.array_equal(res.neighbors_row_splits.cpu().numpy(), rs)
    assert np.array_equal(host_ids(res.neighbors_index, n), idx)
    assert np.array_equal(res.neighbors_distance.cpu().numpy(), d, equal_nan=True)


@pytest.mark.parametrize("name", list(E.BUILDERS))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_radius_searches_bit_equal_to_oracle(name, metric, ignore):
    c = E.case(name)
    p, q, ps, qs, radii = device_case(name)
    m = S.METRICS[metric]
    fixed = S.c_search_radius(c.points, c.queries, c.radius, None, c.ps, c.qs, m, ignore)
    per_query = S.c_search_radius(c.points, c.queries, 0.0, c.radii, c.ps, c.qs, m, ignore, ignore)
    for index_dtype in INDEX_DTYPES:
        res = M.ops.fixed_radius_search(p, q, c.radius, ps, qs, index_dtype=index_dtype, metric=metric,
                                        ignore_query_point=ignore)
        check_radius(res, fixed, len(c.points), index_dtype)
        res = M.ops.radius_search(p, q, radii, ps, qs, index_dtype=index_dtype, metric=metric,
                                  ignore_query_point=ignore, return_distances=True, normalize_distances=ignore)
        check_radius(res, per_query, len(c.points), index_dtype)


def test_knn_raw_l2_path_on_nonfinite_input():
    """knn_search_raw (o3dml_knn_search, the dense L2 rows RandLA-Net gathers with): a row that finds fewer than k
    rankable points is padded with -1 / +inf, never with an out-of-range id; +inf distances are ranked."""
    c = E.case("nonfinite")
    p, q, ps, qs, _ = device_case("nonfinite")
    k = 16
    ref_idx, ref_d, ref_n = ref_knn("nonfinite", k, "L2", False)
    assert (ref_n < k).any() and np.isposinf(ref_d[ref_idx >= 0]).any()
    for index_dtype in INDEX_DTYPES:
        idx = torch.full((len(c.queries), k), -7, dtype=index_dtype, device="cuda")
        d2 = torch.full((len(c.queries), k), -7.0, dtype=torch.float32, device="cuda")
        M.ops.knn_search_raw(p, ps, q, qs, k, idx, d2)
        assert np.array_equal(host_ids(idx, len(c.points)), ref_idx)
        assert np.array_equal(d2.cpu().numpy(), ref_d)


def test_knn_search_still_refuses_items_smaller_than_k():
    p, q, ps, qs, _ = device_case("kedges")
    with pytest.raises(RuntimeError, match="fewer than k"):
        M.ops.knn_search(p, q, 9, ps, qs)


@pytest.mark.parametrize("name", ["nonfinite", "far1e7", "batch"])
def test_layers_equal_the_ops(name):
    c = E.case(name)
    p, q, ps, qs, radii = device_case(name)
    k = 8
    kw = dict(metric="L1", ignore_query_point=True, return_distances=True, index_dtype=torch.int64)
    pairs = [(M.ops.FixedRadiusSearch(**kw)(p, q, c.radius, ps, qs),
              M.ops.fixed_radius_search(p, q, c.radius, ps, qs, **kw)),
             (M.ops.RadiusSearch(normalize_distances=True, **kw)(p, q, radii, ps, qs),
              M.ops.radius_search(p, q, radii, ps, qs, normalize_distances=True, **kw))]
    if not E.short_items(c, k):
        pairs.append((M.ops.KNNSearch(**kw)(p, q, k, ps, qs), M.ops.knn_search(p, q, k, ps, qs, **kw)))
    for a, b in pairs:
        for x, y in zip(a, b):
            assert torch.equal(x.isnan(), y.isnan()) and torch.equal(x.nan_to_num(), y.nan_to_num())
    ref = S.c_search_radius(c.points, c.queries, c.radius, None, c.ps, c.qs, 1, True)
    check_radius(pairs[0][0], ref, len(c.points), torch.int64)
