"""The voxelisation and grid-subsampling oracles (oracle/ops_ref.c, oracle/ops.py) against the float64 partition of
tests/voxel_cases.py, at range edges, batch edges and adversarial cloud minima; the subsample grid origin; and the
refusals of o3dml_voxelize for grids it cannot build.  Needs no GPU."""
import numpy as np
import pytest

from oracle import ops as O
from open3d_ml_b200 import _lib as L
import voxel_cases as V


@pytest.mark.parametrize("grid", sorted(V.GRIDS))
def test_voxelize_oracles_partition_range_edges(grid):
    g = V.GRIDS[grid]
    pts = V.range_edge_cloud(g, 11)
    splits = V.ragged_splits([len(pts)])
    c = O.c_voxelize(pts, splits, *g)
    nres = O.np_voxelize(pts, splits, *g)
    for k in c:
        assert np.array_equal(c[k], nres[k]), k
    part = V.check_partition(c, pts, splits, *g)
    # p == rmax is kept, its index at most the extent (DESIGN.md section 2); an ulp outside either bound is not
    at_max = np.nonzero(np.all(pts == V.f32(g[2]), 1))[0]
    assert len(at_max) and part["inside"][at_max].all()
    assert (c["voxel_coords"] <= V.grid_extent(*g)).all()
    vs, lo, hi = (V.f32(a) for a in g)
    outside = np.any((pts < lo) | (pts > hi) | ~np.isfinite(pts), 1)
    assert not part["inside"][outside].any() and part["inside"][~outside].all()


@pytest.mark.parametrize("batch", [1, 255, 256, 257, 1000])
def test_voxelize_oracle_batch_edges_and_caps(batch):
    g = V.GRIDS["fine3d"]
    lens = V.batch_lens(batch, batch)
    splits = V.ragged_splits(lens)
    pts = V.cloud_in(g, int(splits[-1]), batch, margin=0.5)
    c = O.c_voxelize(pts, splits, *g)
    part = V.check_partition(c, pts, splits, *g)
    per_item = np.diff(c["voxel_batch_splits"])
    top = int(per_item.max())
    for cap in (top - 1, top, top + 1):
        if cap < 1:
            continue
        got = O.c_voxelize(pts, splits, *g, max_voxels=cap)
        nres = O.np_voxelize(pts, splits, *g, max_voxels=cap)
        for k in got:
            assert np.array_equal(got[k], nres[k]), k
        assert np.array_equal(np.diff(got["voxel_batch_splits"]), np.minimum(per_item, cap))
        V.check_partition(got, pts, splits, *g, max_voxels=cap)
    assert part["inside"].sum() == len(c["voxel_point_indices"])


@pytest.mark.parametrize("dl", V.DLS)
def test_subsample_range_origin_is_at_or_below_the_minimum(dl):
    """origin <= min on every axis, and min - origin < dl up to one float32 spacing of the origin (rounding the origin
    down to float32 can move it that far below floor(min / dl) * dl)."""
    mins = V.adversarial_minima(dl, 40, 1)
    assert len(mins) >= 3
    assert (V.rounded_origin32(mins, dl) > mins).all()       # the float32 product lands above every one of these
    rng = np.random.default_rng(int(dl * 1000))
    rand = rng.uniform(-100, 100, 4000).astype(np.float32)
    vals = np.concatenate([mins, rand])
    for m in vals[:len(vals) // 3 * 3].reshape(-1, 3):
        origin, mx = O.subsample_range(m[None, :], dl)
        o64, m64 = origin.astype(np.float64), m.astype(np.float64)
        assert (o64 <= m64).all(), (m, origin)
        assert (m64 - o64 < np.float64(np.float32(dl)) + np.spacing(np.abs(origin)).astype(np.float64)).all()
        assert np.array_equal(mx, m)


def test_subsample_range_refuses_non_finite_points():
    pts = np.zeros((10, 3), np.float32)
    for v in (np.nan, np.inf, -np.inf):
        bad = pts.copy()
        bad[4, 1] = v
        with pytest.raises(RuntimeError):
            O.subsample_range(bad, 0.1)


@pytest.mark.parametrize("dl", V.DLS)
def test_subsample_oracles_keep_adversarial_minima(dl):
    """Every point of a cloud whose minimum is an adversarial value on each axis lands in exactly one voxel, and both
    subsampling restatements give the float64 voxel count."""
    pts, mins = V.adversarial_cloud(dl, 5)
    lens = [1000, 0, len(pts) - 1000]
    splits = V.ragged_splits(lens)
    origin, mx = O.subsample_range(pts, dl)
    assert (origin <= mins).all()
    vox = O.c_voxelize(pts, splits, [dl] * 3, origin, mx)
    part = V.check_partition(vox, pts, splits, [dl] * 3, origin, mx)
    assert part["inside"].all()
    a = O.c_subsample_batch(pts, lens, None, None, dl)
    b = O.np_subsample_batch(pts, lens, None, None, dl)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert np.array_equal(a[1], np.diff(vox["voxel_batch_splits"]))


def test_oracle_voxel_reduce_against_float64():
    """Mean within the sequential-sum bound, max and first exact, NaN kept by all three, majority labels with ties to
    the smallest (negative labels, single-label voxels)."""
    rng = np.random.default_rng(9)
    n = 6000
    pts = (rng.random((n, 3)) * [4, 3, 2] - [40, 1, 1]).astype(np.float32)
    feats = (rng.standard_normal((n, 4)) * [1, 100, 1e-3, 1]).astype(np.float32)
    feats[rng.integers(0, n, 5), 3] = np.nan
    labs = rng.integers(-3, 3, n).astype(np.int32)
    labs[pts[:, 0] < -39.5] = 7                    # whole voxels of one label
    origin, mx = O.subsample_range(pts, 0.25)
    vox = O.c_voxelize(pts, None, [0.25] * 3, origin, mx)
    vrs, pidx = vox["voxel_point_row_splits"], vox["voxel_point_indices"]
    for pm, fm, name in ((0, 0, "mean"), (1, 1, "max"), (2, 2, "first")):
        op, of, ol = V.oracle_reduce(pts, feats, labs, vrs, pidx, pm, fm)
        for got, src in ((op, pts), (of, feats)):
            ref = V.np_reduce64(src, vrs, pidx, name)
            nan = np.isnan(ref)
            assert np.array_equal(np.isnan(got), nan)
            if name == "mean":
                assert (np.abs(got[~nan] - ref[~nan]) <= V.mean_bound(src, vrs, pidx)[~nan]).all()
            else:
                assert np.array_equal(got[~nan].astype(np.float64), ref[~nan])
        assert np.array_equal(ol, V.majority64(labs, vrs, pidx))
    assert (V.majority64(labs, vrs, pidx) < 0).any() and (V.majority64(labs, vrs, pidx) == 7).any()
    assert np.isnan(of).any()


# ---------------------------------------------------------------------------------------- o3dml_voxelize refusals
HOST_WORD = np.zeros(1, np.int64)


def refusal(vs, rmin, rmax, batch=1):
    """(status, message, launches) of o3dml_voxelize on a host-side grid with NULL device pointers and no workspace:
    the grid is checked before anything is enqueued."""
    h = [np.asarray(a, np.float32) for a in (vs, rmin, rmax)]
    n0 = L.lib().o3dml_launch_count()
    rc = L.lib().o3dml_voxelize(None, 1000, 3, None, batch, h[0].ctypes.data, h[1].ctypes.data, h[2].ctypes.data, 32,
                                1000, None, None, None, None, None, None, None, 0, None)
    return rc, L.lib().o3dml_last_error().decode(), L.lib().o3dml_launch_count() - n0


@pytest.mark.parametrize("vs,rmin,rmax", [
    ([1, 1, 1e-12], [0, 0, 0], [1000, 1000, 10]),           # the last extent alone overflows int64 products
    ([1, 1, 1], [0, 0, 0], [1e6, 1e6, 1e6]),                # 10^12 cells after two axes, 10^18 after the third
    ([1, 1, 1], [0, 0, 0], [2e12, 1, 1]),                   # one extent beyond 2^40
])
def test_voxelize_refuses_a_grid_over_2_40_cells(vs, rmin, rmax):
    rc, msg, launches = refusal(vs, rmin, rmax)
    assert rc == 1 and "grid too large" in msg and launches == 0, (rc, msg)


@pytest.mark.parametrize("vs,rmin,rmax", [
    ([1, 1, 1], [0, 0, 0], [np.inf, 1, 1]),
    ([1, 1, 1], [0, -np.inf, 0], [1, 1, 1]),
    ([1, 1, 1], [0, 0, np.nan], [1, 1, 1]),
    ([1, 1, 1], [0, 0, 0], [1, np.nan, 1]),
    ([1, 1e-45, 1], [0, 0, 0], [1, 1, 1]),                 # 1 / vs overflows to inf
])
def test_voxelize_refuses_a_non_finite_grid(vs, rmin, rmax):
    rc, msg, launches = refusal(vs, rmin, rmax)
    assert rc == 1 and "finite grid" in msg and launches == 0, (rc, msg)


def test_voxelize_grid_at_the_cell_limit_reaches_the_workspace_check():
    """2^40 cells exactly is a grid: the call gets as far as the workspace refusal."""
    rc, msg, launches = refusal([1, 1, 1], [0, 0, 0], [2 ** 20 - 1, 2 ** 19 - 1, 0.5])   # (2^20, 2^19, 2) cells
    assert rc == 2 and "workspace too small" in msg and launches == 0, (rc, msg)
