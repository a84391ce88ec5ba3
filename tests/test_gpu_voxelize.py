"""voxelize (voxelize.cu: hash, stable radix sort and scan of prims.cu, segment, emit), grid subsampling, voxel pooling
and voxel_reduce (subsample.cu) against the float64 partition of tests/voxel_cases.py.  Every voxelize case is checked
three ways: bit-equal to the C oracle (c_voxelize / c_subsample_batch); every point off the band in its float64 voxel;
with no caps binding, every finite in-range point listed exactly once and the voxel count equal to the float64 count."""
import numpy as np
import pytest
import torch

from oracle import ops as O
from open3d_ml_b200 import synth
import open3d_ml_b200 as M
import helpers as H
import voxel_cases as V

pytestmark = pytest.mark.gpu
INT64_MAX = 2 ** 63 - 1


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_voxelize(pts, splits, grid, max_pts=None, max_vox=None):
    """voxelize_raw with the batch ids: (result dict of numpy arrays, voxel_batch_id)."""
    coords, pidx, vrs, bsp, bid, counts = M.ops.voxelize_raw(
        T(V.f32(pts)[:, :3]), T(np.asarray(splits, np.int64)), grid[0], grid[1], grid[2],
        max_pts or INT64_MAX, max_vox or INT64_MAX, want_batch_id=True)
    m, kept = (int(v) for v in counts.tolist())
    res = dict(voxel_coords=coords[:m].cpu().numpy(), voxel_point_indices=pidx[:kept].cpu().numpy(),
               voxel_point_row_splits=vrs[:m + 1].cpu().numpy(), voxel_batch_splits=bsp.cpu().numpy())
    return res, bid[:m].cpu().numpy()


def check3(pts, splits, grid, max_pts=None, max_vox=None, binding=None):
    """Bit-equal to c_voxelize, and the float64 partition (conservation only when no cap binds)."""
    res, bid = gpu_voxelize(pts, splits, grid, max_pts, max_vox)
    ref = O.c_voxelize(V.f32(pts)[:, :3], splits, *grid, max_pts or 2 ** 62, max_vox or 2 ** 62)
    for k in ref:
        assert np.array_equal(res[k], ref[k]), k
    binding = (max_pts is not None or max_vox is not None) if binding is None else binding
    part = V.check_partition(res, pts, splits, *grid, max_points=max_pts if binding else None,
                             max_voxels=max_vox if binding else None, batch_id=bid)
    return res, part


# ------------------------------------------------------------------------------------------------ 1. range edges
@pytest.mark.parametrize("grid", sorted(V.GRIDS))
def test_voxelize_range_edges(grid):
    """Points exactly at rmin and rmax (kept, index == extent possible), an ulp outside either bound, +-0.0, NaN and
    +-inf in each axis, on LiDAR ranges with negative minima and +-150 m at 0.05 and 0.16 m."""
    g = V.GRIDS[grid]
    pts = V.range_edge_cloud(g, 3)
    res, part = check3(pts, V.ragged_splits([len(pts)]), g)
    vs, lo, hi = (V.f32(a) for a in g)
    outside = np.any((pts < lo) | (pts > hi) | ~np.isfinite(pts), 1)
    assert not part["inside"][outside].any() and part["inside"][~outside].all()
    assert (res["voxel_coords"] <= V.grid_extent(*g)).all()


# ------------------------------------------------------------------------------------------- 2. scheduling edges
@pytest.mark.parametrize("n", V.sched_sizes())
def test_voxelize_radix_and_scan_tile_edges(n):
    """n at 1 and at 2048 k +- 1 (radix tile), 4096 k +- 1 (scan tile) for k = 1, 2, 16, and 65 537."""
    g = V.GRIDS["kitti"]
    pts = V.cloud_in(g, n, n, margin=2.0)
    pts[n // 2:] = pts[: n - n // 2]                        # shared voxels, duplicate ids in the sort
    check3(pts, V.ragged_splits([n]), g)
    if n > 4:
        check3(pts, V.ragged_splits([n // 3, 0, n - n // 3]), g, max_pts=3, max_vox=n // 50 + 1)


def test_voxelize_waymo_batch_of_eight_frames():
    """1.44 M points in 8 Waymo-sized frames: the look-back scan runs over about 350 tiles."""
    g = V.GRIDS["waymo"]
    frames = [synth.lidar_frame(180000, 40 + i, synth.WAYMO_RANGE, with_intensity=False) for i in range(8)]
    pts = np.concatenate(frames)
    res, _ = check3(pts, V.ragged_splits([len(f) for f in frames]), g)
    assert len(pts) == 1440000 and len(res["voxel_point_indices"]) == len(pts)
    check3(pts, V.ragged_splits([len(f) for f in frames]), g, max_pts=20, max_vox=32000)


@pytest.mark.parametrize("passes", sorted(V.PASS_GRIDS))
def test_voxelize_radix_pass_counts(passes):
    """Grids and batch sizes whose keys need 1, 2, 3, 5 and 8 radix passes."""
    g, batch = V.PASS_GRIDS[passes]
    assert V.radix_passes(*g, batch) == passes
    rng = np.random.default_rng(passes)
    n = 20000
    lens = np.bincount(rng.integers(0, batch, n), minlength=batch) if batch > 1 else np.array([n])
    pts = V.cloud_in(g, n, passes, margin=0.1)
    vs, lo, hi = (np.asarray(a, np.float64) for a in g)
    pts[::2] = (lo + (np.floor((pts[::2] - lo) / (hi - lo) * 4) + 0.5) * (hi - lo) / 4).astype(np.float32)
    check3(pts, V.ragged_splits(lens), g)


# ------------------------------------------------------------------------------------------------- 3. stability
def test_voxelize_ten_thousand_points_in_one_voxel_across_radix_tiles():
    """Every third of 30 000 points falls in one voxel: its ids ascend across 15 radix tiles, and a
    max_points_per_voxel cap keeps the smallest ids."""
    g = V.GRIDS["kitti"]
    rng = np.random.default_rng(7)
    pts = V.cloud_in(g, 30000, 7)
    one = np.arange(0, 30000, 3)
    corner = np.array([62 * 0.16, -39.68 + 216 * 0.16, -1.0])       # cell (62, 216, 0), 0.01 m inside its faces
    pts[one] = (corner + rng.uniform(0.01, 0.15, (len(one), 3)) * [1, 1, 0]).astype(np.float32)
    splits = V.ragged_splits([30000])
    res, part = check3(pts, splits, g)
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    v = int(np.nonzero(pidx[vrs[:-1]] == 0)[0][0])
    assert np.array_equal(pidx[vrs[v]:vrs[v + 1]], one)
    res, _ = check3(pts, splits, g, max_pts=37)
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    v = int(np.nonzero(pidx[vrs[:-1]] == 0)[0][0])
    assert np.array_equal(pidx[vrs[v]:vrs[v + 1]], one[:37])


def test_voxelize_duplicates_of_one_point():
    g = V.GRIDS["fine3d"]
    pts = V.cloud_in(g, 9000, 8)
    pts[1000:6000] = pts[17]
    splits = V.ragged_splits([9000])
    res, _ = check3(pts, splits, g)
    res, _ = check3(pts, splits, g, max_pts=5)
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    v = int(np.nonzero(pidx[vrs[:-1]] == 17)[0][0])
    assert list(pidx[vrs[v]:vrs[v + 1]]) == [17, 1000, 1001, 1002, 1003]


# ---------------------------------------------------------------------------------------------- 4. batch edges
@pytest.mark.parametrize("batch", [1, 255, 256, 257, 1000])
def test_voxelize_batch_edges_caps_and_batch_ids(batch):
    """vox_batch_bounds_kernel strides over 256 threads; empty items first, last and in a run; max_voxels at an item's
    count - 1, count and count + 1; voxel_batch_id against the float64 item."""
    g = V.GRIDS["fine3d"]
    lens = V.batch_lens(batch, batch)
    splits = V.ragged_splits(lens)
    pts = V.cloud_in(g, int(splits[-1]), batch, margin=0.5)
    res, _ = check3(pts, splits, g)
    per_item = np.diff(res["voxel_batch_splits"])
    top = int(per_item.max())
    counts = sorted({top, int(np.median(per_item[per_item > 0]))})
    for c in counts:
        for cap in (c - 1, c, c + 1):
            if cap >= 1:
                got, _ = check3(pts, splits, g, max_vox=cap, binding=cap < top)
                assert np.array_equal(np.diff(got["voxel_batch_splits"]), np.minimum(per_item, cap))


# --------------------------------------------------------------------------- 5. subsample, pooling and the pyramid
def check_reduce(got_pts, got_feats, got_labs, pts, feats, labs, vrs, pidx, pos="mean", feat="mean"):
    """Per-voxel outputs against float64 over the given voxel lists: mean within mean_bound, max / first exact,
    labels the majority with ties to the smallest.  The means' largest |error| / bound measured on an H100 80GB HBM3
    (700 W power limit) over this file: 0.665 (subsample at dl = 0.3), 0.658 (voxel_reduce)."""
    for got, src, mode in ((got_pts, pts, pos), (got_feats, feats, feat)):
        if got is None:
            continue
        got = np.asarray(got, np.float64)
        ref = V.np_reduce64(src, vrs, pidx, mode)
        nan = np.isnan(ref)
        assert np.array_equal(np.isnan(got), nan)
        if mode == "mean":
            bound = V.mean_bound(src, vrs, pidx)
            err = np.abs(got - ref)[~nan]
            assert (err <= bound[~nan]).all()
        else:
            assert np.array_equal(got[~nan], ref[~nan])
    if got_labs is not None:
        assert np.array_equal(np.asarray(got_labs, np.int64), V.majority64(labs, vrs, pidx))


def subsample_partition(pts, lens, dl):
    """The grid the library subsamples on, voxelized and checked against float64: every point inside."""
    origin, mx = M.ops._subsample_range(T(pts), dl)
    o_ref, mx_ref = O.subsample_range(pts, dl)
    assert np.array_equal(origin, o_ref) and np.array_equal(mx, mx_ref)
    assert (origin <= pts.min(0)).all()
    res, part = check3(pts, V.ragged_splits(lens), ([dl] * 3, origin, mx))
    assert part["inside"].all()
    return res, origin


@pytest.mark.parametrize("dl", V.DLS)
def test_subsample_keeps_adversarial_minima(dl):
    """A cloud whose minimum on each axis is a value at which floor(min / dl) * dl rounds above it in float32: every
    point lands in one voxel, subsample_batch / subsample are bit-equal to the oracle, counts equal the float64 ones,
    barycentres / feature means within the sequential-sum bound of float64, labels the majority."""
    pts, mins = V.adversarial_cloud(dl, 5)
    n = len(pts)
    rng = np.random.default_rng(int(dl * 1000))
    feats = (rng.standard_normal((n, 4)) * [1, 50, 1e-3, 1]).astype(np.float32)
    labs = rng.integers(-2, 4, n).astype(np.int64)
    lens = [1000, 0, n - 1000]
    res, origin = subsample_partition(pts, lens, dl)
    got = M.subsample_batch(pts, lens, features=feats, classes=labs, sampleDl=dl)
    ref = O.c_subsample_batch(pts, lens, feats, labs, dl)
    for a, b in zip(got, ref):
        assert np.array_equal(np.asarray(a).astype(b.dtype), b)
    assert np.array_equal(got[1], np.diff(res["voxel_batch_splits"]))
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    check_reduce(got[0], got[2], got[3], pts, feats, labs, vrs, pidx)
    one = M.subsample(pts, features=feats, classes=labs.astype(np.int32), sampleDl=dl)
    ref1 = O.c_subsample_batch(pts, [n], feats, labs, dl)
    for a, b in zip(one, (ref1[0], ref1[2], ref1[3])):
        assert np.array_equal(np.asarray(a).astype(b.dtype), b)
    assert len(one[0]) == len(subsample_partition(pts, [n], dl)[0]["voxel_coords"])


@pytest.mark.parametrize("position_fn", ["average", "nearest_neighbor", "center"])
@pytest.mark.parametrize("feature_fn", ["average", "max", "nearest_neighbor"])
def test_voxel_pooling_on_adversarial_minima(position_fn, feature_fn):
    dl = 0.05
    pts, _ = V.adversarial_cloud(dl, 6)
    rng = np.random.default_rng(6)
    feats = rng.standard_normal((len(pts), 5)).astype(np.float32)
    feats[3, 1] = np.nan
    res, origin = subsample_partition(pts, [len(pts)], dl)
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    m = len(res["voxel_coords"])
    r = M.ops.voxel_pooling(torch.from_numpy(pts), torch.from_numpy(feats), dl, position_fn, feature_fn)
    gp, gf = r.pooled_positions.numpy().astype(np.float64), r.pooled_features.numpy()
    assert gp.shape == (m, 3) and gf.shape == (m, 5)
    centre = (res["voxel_coords"] + 0.5) * np.float64(np.float32(dl)) + origin.astype(np.float64)
    if "nearest_neighbor" in (position_fn, feature_fn):
        # The member nearest the voxel centre.  The library ranks by float32 d2 from a float32 centre, so the member
        # it takes may lie farther (float64) than the nearest by up to the centre's rounding, 2 u |c| per axis, times
        # 2 |p - c| <= 2 sqrt(3) dl over three axes, plus three roundings of d2 <= 3 dl^2 (3.8e-6 m^2 here).  Measured
        # on an H100 80GB HBM3 (700 W power limit): 0, the float64-nearest member was always the one taken.
        tol = 3 * 2 * np.sqrt(3) * dl * 2 * V.U * np.abs(centre).max() + 3 * V.U * 3 * dl * dl
        for v in range(m):
            rows = pidx[vrs[v]:vrs[v + 1]]
            d2 = ((pts[rows].astype(np.float64) - centre[v]) ** 2).sum(1)
            near = rows[d2 <= d2.min() + tol]
            if position_fn == "nearest_neighbor":
                hit = near[(pts[near] == gp[v]).all(1)]
            else:
                hit = near[np.all((feats[near] == gf[v]) | (np.isnan(feats[near]) & np.isnan(gf[v])), 1)]
            assert len(hit), "voxel %d: the pooled point is not among its nearest members" % v
            if position_fn == "nearest_neighbor" and feature_fn == "nearest_neighbor":
                assert any(np.array_equal(feats[h], gf[v], equal_nan=True) for h in hit)
    if position_fn == "average":
        check_reduce(gp, None, None, pts, None, None, vrs, pidx)
    if position_fn == "center":
        # (coords + 0.5) * dl + origin in float32: at most three roundings of values up to |centre| (61.8 m here, a
        # bound of 1.1e-5 m).  Measured on an H100 80GB HBM3 (700 W power limit): 1.6e-6 m.
        assert np.abs(gp - centre).max() <= 3 * V.U * np.abs(centre).max()
    if feature_fn in ("average", "max"):
        check_reduce(None, gf, None, None, feats, None, vrs, pidx, feat="mean" if feature_fn == "average" else "max")


def test_kpfcnn_pyramid_on_adversarial_minima():
    """KPFCNN segmentation_inputs (kpconv.build_batch) on clouds shifted so that the batch minimum of every axis is an
    adversarial value of the first subsampling dl: each level's point count per item equals the float64 partition's
    of the level below."""
    from open3d_ml_b200.kpconv import build_batch
    _, extra = H.state_dict("kpconv_s3dis.manifest.json", 5)
    cfg = extra["cfg"]
    r = cfg["first_subsampling_dl"] * cfg["conv_radius"]
    dl0 = 2 * r / cfg["conv_radius"]
    mins = V.adversarial_minima(dl0, 3, 2).astype(np.float64)
    clouds = [synth.room_cloud(9000, 80, room=(3.0, 2.5, 2.0)), synth.room_cloud(6000, 81, room=(3.0, 2.5, 2.0))]
    lo = np.min([c[0].min(0) for c in clouds], axis=0).astype(np.float64)
    clouds = [((c[0].astype(np.float64) - lo + mins).astype(np.float32), c[1]) for c in clouds]
    P = np.concatenate([c[0] for c in clouds])
    assert np.array_equal(P.min(0), mins.astype(np.float32))
    assert (V.rounded_origin32(P.min(0), dl0) > P.min(0)).all()
    b = build_batch(clouds, cfg)
    for lvl in range(cfg["num_layers"] - 1):
        P = b["points"][lvl].cpu().numpy()
        lens = b["lengths"][lvl].cpu().numpy().astype(np.int64)
        res, _ = subsample_partition(P, lens, 2 * r / cfg["conv_radius"])
        assert np.array_equal(b["lengths"][lvl + 1].cpu().numpy(), np.diff(res["voxel_batch_splits"]))
        r *= 2


# ------------------------------------------------------------------------------------ 6. voxel_reduce vs float64
def test_voxel_reduce_against_float64_through_strided_inputs():
    """Mean / max / first of positions and features read through row strides larger than their channel counts (the
    C ABI's point_stride and feat_stride), labels with negative values and single-label voxels, NaN features: all
    against float64 over the float64-checked voxel lists, and bit-equal to oracle_voxel_reduce."""
    rng = np.random.default_rng(12)
    n, F = 8000, 6
    base = np.empty((n, 5), np.float32)
    base[:, :3] = (rng.random((n, 3)) * [4, 3, 2] - [40, 1, 1]).astype(np.float32)
    base[:, 3:] = 7.0
    fbase = (rng.standard_normal((n, F + 3)) * 10).astype(np.float32)
    fbase[:, 2] *= 1e3
    fbase[rng.integers(0, n, 6), 4] = np.nan
    labs = rng.integers(-4, 3, n).astype(np.int32)
    labs[base[:, 0] < -39.6] = -9
    pts, feats = base[:, :3], fbase[:, :F]
    res, _ = subsample_partition(np.ascontiguousarray(pts), [n], 0.2)
    vrs, pidx = res["voxel_point_row_splits"], res["voxel_point_indices"]
    m = len(res["voxel_coords"])
    tp, tf = T(base)[:, :3], T(fbase)[:, :F]
    assert tp.stride(0) == 5 and tf.stride(0) == F + 3
    for mode, name in ((0, "mean"), (1, "max"), (2, "first")):
        op, of, ol = M.ops.voxel_reduce(tp, tf, T(labs), T(vrs), T(pidx), None, m, position_mode=mode,
                                        feature_mode=mode)
        op, of, ol = op.cpu().numpy(), of.cpu().numpy(), ol.cpu().numpy()
        check_reduce(op, of, ol, pts, feats, labs, vrs, pidx, pos=name, feat=name)
        assert np.isnan(of[:, 4]).any()
        rp, rf, rl = V.oracle_reduce(pts, feats, labs, vrs, pidx, mode, mode)
        assert np.array_equal(op, rp) and np.array_equal(of, rf, equal_nan=True) and np.array_equal(ol, rl)
    maj = V.majority64(labs, vrs, pidx)
    assert (maj < 0).any() and (maj == -9).any()
