"""Voxelisation and grid-subsampling cases shared by tests/test_gpu_voxelize.py (voxelize.cu with the radix sort and scan
of prims.cu, subsample.cu) and tests/test_oracle_voxelize.py (oracle/ops_ref.c, oracle/ops.py), and the float64
partition both are held to: every finite point with rmin <= p <= rmax lands in exactly one voxel,
floor((p - rmin) / vs) per axis, inside its own batch item.
Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
import numpy as np

F32 = np.float32
U = 2.0 ** -24          # unit roundoff of float32

# The band in which a float32 voxel index may legitimately differ from the float64 one.  The kernels compute
# q = (int)(fl(fl(p - rmin) * fl(1 / vs))).  With x = (p - rmin) / vs exact, each of the three roundings has relative
# error at most u = 2^-24, so q_real = x (1 + d1)(1 + d2)(1 + d3) and |q_real - x| <= ((1 + u)^3 - 1) x < 3.0000001 u x.
# floor(q_real) differs from floor(x) only when x lies within that distance of an integer, a voxel face.  BAND_REL =
# 4 u covers it with room for the one rounding of the float64 evaluation of x (relative 2^-53).  A point with
# x = 0 (p == rmin) is exact in both and never in the band.
BAND_REL = 4 * U

# Voxel sizes of the subsampling cases: the KPConv pyramid's 0.04 .. 0.32 m and the sizes between.
DLS = (0.04, 0.05, 0.06, 0.08, 0.1, 0.16, 0.3)

# Grids (voxel size, range min, range max) with negative minima and LiDAR ranges.
GRIDS = {
    "kitti": ([0.16, 0.16, 4.0], [0.0, -39.68, -3.0], [69.12, 39.68, 1.0]),
    "waymo": ([0.32, 0.32, 6.0], [-74.88, -74.88, -2.0], [74.88, 74.88, 4.0]),
    "fine3d": ([0.05, 0.04, 0.03], [-10.0, -8.0, -3.0], [10.0, 8.0, 2.0]),
    "wide005": ([0.05, 0.05, 0.05], [-150.0, -150.0, -150.0], [150.0, 150.0, 150.0]),
    "wide016": ([0.16, 0.16, 0.16], [-150.0, -150.0, -150.0], [150.0, 150.0, 150.0]),
}


def f32(a):
    return np.asarray(a, F32)


def item_of(splits, n):
    """Batch item of every row 0..n-1 (rows outside [splits[0], splits[-1]) get -1)."""
    splits = np.asarray(splits, np.int64)
    it = np.searchsorted(splits, np.arange(n), side="right") - 1
    return np.where((np.arange(n) >= splits[0]) & (np.arange(n) < splits[-1]), it, -1)


def partition64(points, splits, voxel_size, rmin, rmax):
    """The float64 partition of points [N, >=3] (splits int64 [B+1]) on the grid (voxel_size, rmin, rmax), all taken at
    their float32 values.  Returns a dict of
      inside [N] bool   finite, rmin <= p <= rmax on every axis, and inside a batch item
      item   [N] int64  batch item (-1 outside every item)
      ijk    [N,3] int64  floor((p - rmin) / vs) (0 where not inside)
      face   [N] float64  distance from x = (p - rmin) / vs to the nearest voxel face, in cells (min over axes)
      band   [N] bool   inside and within BAND_REL * x of a face on some axis"""
    p = f32(points)[:, :3].astype(np.float64)
    n = len(p)
    vs, lo, hi = (f32(a).astype(np.float64) for a in (voxel_size, rmin, rmax))
    item = item_of(splits if splits is not None else [0, n], n)
    with np.errstate(invalid="ignore"):
        inside = np.all((p >= lo) & (p <= hi), axis=1) & (item >= 0)
        x = np.where(inside[:, None], (p - lo) / vs, 0.0)
    ijk = np.floor(x).astype(np.int64)
    frac = x - ijk
    dist = np.minimum(frac, 1.0 - frac)
    band = inside & np.any(dist < BAND_REL * x, axis=1)
    return dict(inside=inside, item=item, ijk=ijk, face=dist.min(axis=1), band=band)


def grid_extent(voxel_size, rmin, rmax):
    """Per-axis extent as the library computes it: ceil(fl(fl(max - min) * fl(1 / vs))), at least 1."""
    vs, lo, hi = f32(voxel_size), f32(rmin), f32(rmax)
    c = ((hi - lo).astype(F32) * (F32(1) / vs).astype(F32)).astype(F32)
    return np.maximum(np.ceil(c), 1).astype(np.int64)


def radix_passes(voxel_size, rmin, rmax, batch):
    """8-bit radix passes the voxel sort makes: the keys run up to cells * batch (the out-of-range key)."""
    cells = int(np.prod(grid_extent(voxel_size, rmin, rmax) + 1))
    bits = max((cells * batch).bit_length(), 1)
    return (bits + 7) // 8


def check_partition(res, points, splits, voxel_size, rmin, rmax, max_points=None, max_voxels=None, batch_id=None):
    """A voxelize result (numpy dict with voxel_coords, voxel_point_indices, voxel_point_row_splits,
    voxel_batch_splits) against the float64 partition:
      * every listed point is inside, in its float64 item, and, outside the band, in its float64 voxel; inside the
        band within one cell of it;
      * voxels of an item ascend in linear index and hold ascending point ids;
      * with no caps binding: every inside point is listed exactly once and the voxel count equals the float64 count
        (band points counted in the voxel the kernel chose, which the first check bounds).
    Returns the partition."""
    pts = f32(points)
    n = len(pts)
    part = partition64(pts, splits, voxel_size, rmin, rmax)
    coords = np.asarray(res["voxel_coords"], np.int64)
    pidx = np.asarray(res["voxel_point_indices"], np.int64)
    vrs = np.asarray(res["voxel_point_row_splits"], np.int64)
    bsp = np.asarray(res["voxel_batch_splits"], np.int64)
    m = len(coords)
    assert len(vrs) == m + 1 and vrs[0] == 0 and vrs[-1] == len(pidx) and bsp[-1] == m
    vox_of = np.repeat(np.arange(m), np.diff(vrs))
    vitem = np.searchsorted(bsp, np.arange(m), side="right") - 1
    if batch_id is not None:
        assert np.array_equal(np.asarray(batch_id, np.int64), vitem)
    assert part["inside"][pidx].all(), "a listed point is outside the range or non-finite"
    assert np.array_equal(part["item"][pidx], vitem[vox_of]), "a point is listed under another batch item"
    diff = coords[vox_of] - part["ijk"][pidx]
    off = ~part["band"][pidx]
    bad = np.nonzero(off & np.any(diff != 0, axis=1))[0]
    assert len(bad) == 0, "points off the band outside their float64 voxel, e.g. %s: face %s, kernel %s, f64 %s" % (
        pidx[bad[:3]], part["face"][pidx[bad[:3]]], coords[vox_of[bad[:3]]], part["ijk"][pidx[bad[:3]]])
    assert np.abs(diff).max(initial=0) <= 1
    ext1 = grid_extent(voxel_size, rmin, rmax) + 1
    lin = coords[:, 0] + ext1[0] * (coords[:, 1] + ext1[1] * coords[:, 2])
    same_item = vitem[1:] == vitem[:-1]
    assert np.all(lin[1:][same_item] > lin[:-1][same_item]), "voxels of an item out of order"
    same_vox = vox_of[1:] == vox_of[:-1]
    assert np.all(pidx[1:][same_vox] > pidx[:-1][same_vox]), "point ids of a voxel out of order"
    if max_points is None and max_voxels is None:
        inside = np.nonzero(part["inside"])[0]
        assert len(pidx) == len(inside) and np.array_equal(np.sort(pidx), inside), \
            "%d inside points, %d listed" % (len(inside), len(pidx))
        ijk = part["ijk"].copy()
        ijk[pidx] = np.where(part["band"][pidx][:, None], coords[vox_of], ijk[pidx])
        keys = np.stack([part["item"][inside], ijk[inside, 0], ijk[inside, 1], ijk[inside, 2]], 1)
        assert len(np.unique(keys, axis=0)) == m
    else:
        counts = np.diff(vrs)
        if max_points is not None:
            assert counts.max(initial=0) <= max_points
        if max_voxels is not None:
            assert np.diff(bsp).max(initial=0) <= max_voxels
    return part


# --------------------------------------------------------------------------------------------------- case builders
def cloud_in(grid, n, seed, margin=0.0):
    """n float32 points uniform in the grid's range, grown by `margin` on every side."""
    vs, lo, hi = (np.asarray(a, np.float64) for a in grid)
    rng = np.random.default_rng(seed)
    return (lo - margin + rng.random((n, 3)) * (hi - lo + 2 * margin)).astype(F32)


def range_edge_cloud(grid, seed, n=4000):
    """Points uniform in range (with 5 % outside), then per axis: exactly at rmin and at rmax, one float32 ulp outside
    either bound, +0.0 and -0.0, NaN, +inf and -inf.  Every special row keeps the other two coordinates in range."""
    vs, lo, hi = (f32(a) for a in grid)
    pts = cloud_in(grid, n, seed, margin=0.05 * float(np.max(hi - lo)))
    rng = np.random.default_rng(seed + 1)
    rows = []
    for d in range(3):
        vals = [lo[d], hi[d], np.nextafter(lo[d], F32(-np.inf)), np.nextafter(hi[d], F32(np.inf)), F32(0.0),
                F32(-0.0), F32(np.nan), F32(np.inf), F32(-np.inf)]
        for v in vals:
            for _ in range(3):
                r = (lo + rng.random(3).astype(F32) * (hi - lo)).astype(F32)
                r[d] = v
                rows.append(r)
    corner = [lo.copy(), hi.copy()]
    pts = np.concatenate([pts, np.stack(rows + corner).astype(F32)])
    return pts[np.random.default_rng(seed + 2).permutation(len(pts))]


def sched_sizes():
    """Point counts at the radix tile (2048 keys) and scan tile (4096 entries) edges of prims.cu, for k = 1, 2, 16."""
    out = {1, 65537}
    for k in (1, 2, 16):
        for t in (2048, 4096):
            out |= {t * k - 1, t * k, t * k + 1}
    return sorted(out)


# Grids whose keys need 1, 2, 3, 5 and 8 radix passes (with the batch given): (voxel size, rmin, rmax), batch.
PASS_GRIDS = {
    1: (([1.0, 1.0, 1.0], [0.0, 0.0, 0.0], [1.0, 1.0, 1.0]), 1),
    2: (([1.0, 1.0, 1.0], [0.0, 0.0, 0.0], [10.0, 10.0, 10.0]), 3),
    3: (([1.0, 1.0, 1.0], [-50.0, -50.0, 0.0], [50.0, 50.0, 10.0]), 2),
    5: (([0.1, 0.1, 0.1], [-100.0, -100.0, -100.0], [100.0, 100.0, 100.0]), 4),
    8: (([1.0, 1.0, 1.0], [0.0, 0.0, 0.0], [10000.0, 10000.0, 10000.0]), 100000),
}


def ragged_splits(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def batch_lens(batch, seed, n_mean=40):
    """Item lengths with empty items first, last and in a run (for batch >= 8)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 2 * n_mean, batch)
    if batch >= 8:
        lens[0] = lens[-1] = 0
        lens[batch // 2: batch // 2 + 5] = 0
    return lens.astype(np.int64)


# ------------------------------------------------------------------------------------------- adversarial minima
def rounded_origin32(m, dl):
    """floor(m / dl) * dl with every operation in float32, rounded to nearest: the formula that can exceed m."""
    m, dl = f32(m), F32(dl)
    return (np.floor((m / dl).astype(F32)) * dl).astype(F32)


def adversarial_minima(dl, count=3, seed=0, lo=-100.0, hi=100.0):
    """Up to `count` float32 minima in [lo, hi] at which rounded_origin32 lands above the minimum, found by a seeded
    search over the float32 values within 8 ulps of k * dl for random integers k (such a minimum sits just below a
    multiple of dl, where float32 m / dl rounds onto the integer).  At least one is always found for DLS."""
    rng = np.random.default_rng(seed + int(round(dl * 1e4)))
    d = F32(dl)
    ks = rng.integers(int(lo / dl), int(hi / dl), 200000).astype(np.float64)
    base = (ks * np.float64(d)).astype(F32)
    cand = [base]
    up, down = base.copy(), base.copy()
    for _ in range(8):
        up, down = np.nextafter(up, F32(np.inf)), np.nextafter(down, F32(-np.inf))
        cand += [up, down]
    c = np.unique(np.concatenate(cand))
    c = c[(c >= lo) & (c <= hi)]
    bad = c[rounded_origin32(c, d) > c]
    return bad[rng.permutation(len(bad))[:count]] if len(bad) else bad


def adversarial_cloud(dl, seed, n=3000, span=(6.0, 5.0, 3.0)):
    """n float32 points whose minimum on axis a is an adversarial minimum of dl (a different one per axis, each held by
    exactly one point), the rest spread over `span` above it."""
    mins = adversarial_minima(dl, 3, seed)
    assert len(mins) == 3, "the search found %d adversarial minima for dl = %g" % (len(mins), dl)
    rng = np.random.default_rng(seed)
    mins = mins.astype(np.float64)
    pts = (mins + 1e-3 + rng.random((n, 3)) * np.asarray(span)).astype(F32)
    for a in range(3):
        pts[a * 7 + 1, a] = F32(mins[a])
    return pts, f32(mins)


def np_reduce64(src, vrs, pidx, mode):
    """Per-voxel float64 mean / max / first of src [N, C] over the CSR lists.  Max and first propagate NaN."""
    src = np.asarray(src, np.float64)
    m = len(vrs) - 1
    out = np.empty((m, src.shape[1]), np.float64)
    for v in range(m):
        rows = src[pidx[vrs[v]:vrs[v + 1]]]
        if mode == "mean":
            out[v] = rows.mean(0)
        elif mode == "max":
            out[v] = np.where(np.isnan(rows).any(0), np.nan, rows.max(0))
        else:
            out[v] = rows[0]
    return out


def mean_bound(src, vrs, pidx):
    """Per-voxel, per-channel bound on |float32 mean - float64 mean|: the sequential float32 sum of c terms errs by at
    most (c - 1) u sum|x| (first order: the k-th partial sum is rounded once, |partial| <= sum|x|), divided by c, plus
    one rounding of the division, u |mean|."""
    src = np.abs(np.asarray(src, np.float64))
    c = np.diff(vrs).astype(np.float64)
    vox = np.repeat(np.arange(len(c)), np.diff(vrs))
    s = np.zeros((len(c), src.shape[1]))
    np.add.at(s, vox, src[pidx])
    return ((c - 1)[:, None] * U * s / c[:, None] + U * s / c[:, None]) * (1 + 1e-6)


def oracle_reduce(points, feats, labels, vrs, pidx, pos_mode, feat_mode):
    """oracle_voxel_reduce (oracle/ops_ref.c) over the CSR lists; modes 0 mean, 1 max, 2 first."""
    import ctypes
    from oracle import ops as O
    points = np.ascontiguousarray(points, F32)
    feats = np.ascontiguousarray(feats, F32)
    F = feats.shape[1]
    labs = None if labels is None else np.ascontiguousarray(labels, np.int32)
    vrs, pidx = np.ascontiguousarray(vrs, np.int64), np.ascontiguousarray(pidx, np.int64)
    m = len(vrs) - 1
    op, of, ol = np.empty((m, 3), F32), np.empty((m, F), F32), np.empty(m, np.int32)

    def p(a, t):
        return a.ctypes.data_as(ctypes.POINTER(t))
    assert O.lib().oracle_voxel_reduce(p(points, ctypes.c_float), 3, p(feats, ctypes.c_float), F,
                                       None if labs is None else p(labs, ctypes.c_int32), p(vrs, ctypes.c_int64),
                                       p(pidx, ctypes.c_int64), ctypes.c_int64(m), pos_mode, feat_mode,
                                       p(op, ctypes.c_float), p(of, ctypes.c_float), p(ol, ctypes.c_int32)) == 0
    return op, of, ol


def majority64(labels, vrs, pidx):
    """Most frequent label per voxel, ties to the smallest."""
    labels = np.asarray(labels, np.int64).reshape(-1)
    out = np.empty(len(vrs) - 1, np.int64)
    for v in range(len(out)):
        vals, cnt = np.unique(labels[pidx[vrs[v]:vrs[v + 1]]], return_counts=True)
        out[v] = vals[np.argmax(cnt)]
    return out
