"""oracle/ops.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU checker for the operator boundary (`open3d.ml.torch.ops` as consumed by the
reference, SURVEY.md section 2.2).  Two independent restatements:

  * ``c_*``  : ctypes bindings of oracle/ops_ref.c (brute force, obviously correct)
  * ``np_*`` : numpy/scipy restatements (lexsort voxelisation, cKDTree candidate
               generation followed by the float32 re-ranking of the contract)

PARITY UNPINNED (see the header of ops_ref.c): the reference's tests hold no
golden vectors for these ops and upstream Open3D is not installable here, so
the two restatements are pinned against each other (tests/test_oracle_ops.py)
and against scipy/sklearn KD-trees, and the contract they implement is written
down in DESIGN.md.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build():
    """Compile oracle/ops_ref.c (gcc) -> oracle/_build/liboracle_ops.so."""
    subprocess.run(["make", "-s", "-C", _HERE], check=True,
                   env={k: v for k, v in os.environ.items() if k not in ("CC", "CXX")})
    return os.path.join(_HERE, "_build", "liboracle_ops.so")


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "_build", "liboracle_ops.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(
                os.path.join(_HERE, "ops_ref.c")):
            build()
        _LIB = ctypes.CDLL(path)
    return _LIB


def _p(a, ty):
    return a.ctypes.data_as(ctypes.POINTER(ty))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _splits(splits, n):
    if splits is None:
        return np.array([0, n], dtype=np.int64)
    return np.ascontiguousarray(splits, dtype=np.int64)


# ----------------------------------------------------------------------------
# C (brute force) oracle
# ----------------------------------------------------------------------------
def c_knn(points, queries, k, points_row_splits=None, queries_row_splits=None):
    """-> (idx int32 [Nq,k] global, d2 float32 [Nq,k]); order (d2, idx) ascending."""
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    idx = np.empty((len(queries), k), np.int32)
    d2 = np.empty((len(queries), k), np.float32)
    rc = lib().oracle_knn(_p(points, ctypes.c_float), _p(ps, ctypes.c_int64),
                          _p(queries, ctypes.c_float), _p(qs, ctypes.c_int64),
                          ctypes.c_int64(len(ps) - 1), ctypes.c_int(k), _p(idx, ctypes.c_int32),
                          _p(d2, ctypes.c_float))
    assert rc == 0
    return idx, d2


def c_radius(points, queries, radius, points_row_splits=None, queries_row_splits=None):
    """-> (neighbors_index int32 [L], row_splits int64 [Nq+1], d2 float32 [L])."""
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    rs = np.zeros(len(queries) + 1, np.int64)
    L = lib()
    args = (_p(points, ctypes.c_float), _p(ps, ctypes.c_int64), _p(queries, ctypes.c_float),
            _p(qs, ctypes.c_int64), ctypes.c_int64(len(ps) - 1), ctypes.c_float(radius),
            _p(rs, ctypes.c_int64))
    assert L.oracle_radius(*args, None, None) == 0
    idx = np.empty(int(rs[-1]), np.int32)
    d2 = np.empty(int(rs[-1]), np.float32)
    assert L.oracle_radius(*args, _p(idx, ctypes.c_int32), _p(d2, ctypes.c_float)) == 0
    return idx, rs, d2


def c_voxelize(points, row_splits, voxel_size, range_min, range_max,
               max_points_per_voxel=2**62, max_voxels=2**62):
    """-> dict(voxel_coords int32 [M,3], voxel_point_indices int64 [L],
    voxel_point_row_splits int64 [M+1], voxel_batch_splits int64 [B+1])."""
    points = _f32(points)
    rs = _splits(row_splits, len(points))
    n = len(points)
    coords = np.empty((max(n, 1), 3), np.int32)
    pidx = np.empty(max(n, 1), np.int64)
    vrs = np.empty(n + 1, np.int64)
    bs = np.empty(len(rs), np.int64)
    m = ctypes.c_int64()
    kept = ctypes.c_int64()
    vs, rmin, rmax = _f32(voxel_size), _f32(range_min), _f32(range_max)
    rc = lib().oracle_voxelize(_p(points, ctypes.c_float), _p(rs, ctypes.c_int64),
                               ctypes.c_int64(len(rs) - 1), _p(vs, ctypes.c_float),
                               _p(rmin, ctypes.c_float), _p(rmax, ctypes.c_float),
                               ctypes.c_int64(int(min(max_points_per_voxel, 2**62))),
                               ctypes.c_int64(int(min(max_voxels, 2**62))),
                               _p(coords, ctypes.c_int32), _p(pidx, ctypes.c_int64),
                               _p(vrs, ctypes.c_int64), _p(bs, ctypes.c_int64),
                               ctypes.byref(m), ctypes.byref(kept))
    assert rc == 0
    M, L = m.value, kept.value
    return dict(voxel_coords=coords[:M].copy(), voxel_point_indices=pidx[:L].copy(),
                voxel_point_row_splits=vrs[:M + 1].copy(), voxel_batch_splits=bs)


# ----------------------------------------------------------------------------
# numpy restatements
# ----------------------------------------------------------------------------
def np_sqdist(q, p):
    """float32 ((dx*dx + dy*dy) + dz*dz), d = q - p, each op rounded once."""
    d = (q.astype(np.float32) - p.astype(np.float32)).astype(np.float32)
    sq = (d * d).astype(np.float32)
    return ((sq[..., 0] + sq[..., 1]).astype(np.float32) + sq[..., 2]).astype(np.float32)


def np_voxelize(points, row_splits, voxel_size, range_min, range_max,
                max_points_per_voxel=2**62, max_voxels=2**62):
    """Sort-based hard voxelisation (contract: ops_ref.c header)."""
    points = _f32(points)
    rs = _splits(row_splits, len(points))
    vs, rmin, rmax = _f32(voxel_size), _f32(range_min), _f32(range_max)
    inv = (np.float32(1.0) / vs).astype(np.float32)
    ext = np.maximum(np.ceil(((rmax - rmin).astype(np.float32) * inv).astype(np.float32)), 1).astype(np.int64)
    coords_out, pidx_out, counts_out, bsplits = [], [], [], [0]
    for b in range(len(rs) - 1):
        ids = np.arange(rs[b], rs[b + 1], dtype=np.int64)
        p = points[ids]
        ok = np.all((p >= rmin) & (p <= rmax), axis=1)
        ids, p = ids[ok], p[ok]
        ijk = (((p - rmin).astype(np.float32)) * inv).astype(np.float32).astype(np.int64)
        h = ijk[:, 0] + (ext[0] + 1) * (ijk[:, 1] + (ext[1] + 1) * ijk[:, 2])
        order = np.lexsort((ids, h))
        h, ids, ijk = h[order], ids[order], ijk[order]
        uniq, first, cnt = np.unique(h, return_index=True, return_counts=True)
        nv = int(min(len(uniq), max_voxels))
        for v in range(nv):
            keep = int(min(cnt[v], max_points_per_voxel))
            pidx_out.append(ids[first[v]:first[v] + keep])
            counts_out.append(keep)
        coords_out.append(ijk[first[:nv]].astype(np.int32).reshape(-1, 3))
        bsplits.append(bsplits[-1] + nv)
    coords = np.concatenate(coords_out) if coords_out else np.zeros((0, 3), np.int32)
    pidx = np.concatenate(pidx_out) if pidx_out else np.zeros((0,), np.int64)
    vrs = np.concatenate([[0], np.cumsum(np.asarray(counts_out, np.int64))]).astype(np.int64)
    return dict(voxel_coords=coords.reshape(-1, 3), voxel_point_indices=pidx,
                voxel_point_row_splits=vrs, voxel_batch_splits=np.asarray(bsplits, np.int64))


def np_ragged_to_dense(values, row_splits, out_col_size, default_value):
    """out[i, j] = values[row_splits[i] + j] for j < min(len_i, out_col_size) else default
    (point_pillars.py:364-366, kpconv.py:2030-2032)."""
    values = np.asarray(values)
    rs = np.asarray(row_splits, np.int64)
    rows = len(rs) - 1
    out = np.empty((rows, out_col_size) + values.shape[1:], values.dtype)
    out[...] = np.asarray(default_value).reshape(-1)[0]
    for i in range(rows):
        n = int(min(rs[i + 1] - rs[i], out_col_size))
        out[i, :n] = values[rs[i]:rs[i] + n]
    return out


def np_knn(points, queries, k, points_row_splits=None, queries_row_splits=None, extra=16):
    """KD-tree candidates re-ranked in float32 by (d2, idx); brute force when a
    candidate set cannot be proven complete."""
    from scipy.spatial import cKDTree
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    idx = np.full((len(queries), k), -1, np.int32)
    d2 = np.full((len(queries), k), np.inf, np.float32)
    for b in range(len(ps) - 1):
        P, Q = points[ps[b]:ps[b + 1]], queries[qs[b]:qs[b + 1]]
        if len(P) == 0 or len(Q) == 0:
            continue
        kk = int(min(len(P), k + extra))
        _, cand = cKDTree(P).query(Q.astype(np.float64), k=kk)
        cand = cand.reshape(len(Q), kk)
        dd = np_sqdist(Q[:, None, :], P[cand])
        order = np.lexsort((cand, dd), axis=1)
        cand_s = np.take_along_axis(cand, order, 1)
        dd_s = np.take_along_axis(dd, order, 1)
        kq = min(k, kk)
        if kk < len(P):
            # incomplete if the worst candidate is not clearly beyond the k-th
            risky = np.nonzero(dd_s[:, -1] <= dd_s[:, kq - 1] * np.float32(1 + 1e-5))[0]
            for r in risky:
                dall = np_sqdist(Q[r][None, :], P)
                o = np.lexsort((np.arange(len(P)), dall))[:kq]
                cand_s[r, :kq], dd_s[r, :kq] = o, dall[o]
        idx[qs[b]:qs[b + 1], :kq] = cand_s[:, :kq] + ps[b]
        d2[qs[b]:qs[b + 1], :kq] = dd_s[:, :kq]
    return idx, d2


def np_radius(points, queries, radius, points_row_splits=None, queries_row_splits=None):
    from scipy.spatial import cKDTree
    points, queries = _f32(points), _f32(queries)
    ps, qs = _splits(points_row_splits, len(points)), _splits(queries_row_splits, len(queries))
    r2 = np.float32(np.float32(radius) * np.float32(radius))
    rows_i, rows_d = [], []
    for b in range(len(ps) - 1):
        P, Q = points[ps[b]:ps[b + 1]], queries[qs[b]:qs[b + 1]]
        if len(Q) == 0:
            continue
        if len(P) == 0:
            rows_i += [np.zeros(0, np.int32)] * len(Q)
            rows_d += [np.zeros(0, np.float32)] * len(Q)
            continue
        cand = cKDTree(P).query_ball_point(Q.astype(np.float64), float(radius) * (1 + 1e-5) + 1e-7)
        for qi, c in enumerate(cand):
            c = np.asarray(c, np.int64)
            dd = np_sqdist(Q[qi][None, :], P[c]) if len(c) else np.zeros(0, np.float32)
            keep = dd <= r2
            c, dd = c[keep], dd[keep]
            o = np.lexsort((c, dd))
            rows_i.append((c[o] + ps[b]).astype(np.int32))
            rows_d.append(dd[o])
    lens = np.array([len(r) for r in rows_i], np.int64)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.concatenate(rows_i) if rows_i else np.zeros(0, np.int32)
    d2 = np.concatenate(rows_d) if rows_d else np.zeros(0, np.float32)
    return idx.astype(np.int32), rs, d2.astype(np.float32)


# ----------------------------------------------------------------------------
# grid subsampling (contract: ops_ref.c, "grid subsampling")
# ----------------------------------------------------------------------------
def subsample_range(points, dl):
    """range_min / range_max of the voxel grid: origin = the largest float32 <= floor(min / dl) * dl, the product
    exact in float64 with dl at its float32 value, so origin <= min; non-finite points raise RuntimeError."""
    points = _f32(points)
    mn, mx = points.min(0), points.max(0)
    if not (np.isfinite(mn).all() and np.isfinite(mx).all()):
        raise RuntimeError("subsample: the points must be finite")
    d = np.float64(np.float32(dl))
    m64 = mn.astype(np.float64)
    k = np.floor(m64 / d)
    k = np.where(k * d > m64, k - 1, k)        # min / d rounded up onto an integer
    o64 = k * d
    origin = o64.astype(np.float32)
    origin = np.where(origin.astype(np.float64) > o64, np.nextafter(origin, np.float32(-np.inf)), origin)
    return origin.astype(np.float32), mx.astype(np.float32)


def c_subsample_batch(points, batches_len, features=None, classes=None, sampleDl=0.1, max_p=0):
    """-> (s_points [M,3], s_len [B] int32, [s_features [M,F]], [s_labels [M] int32])."""
    points = _f32(points)
    rs = np.concatenate([[0], np.cumsum(np.asarray(batches_len, np.int64))]).astype(np.int64)
    origin, mx = subsample_range(points, sampleDl)
    vox = c_voxelize(points, rs, [sampleDl] * 3, origin, mx, 2**62, max_p if max_p > 0 else 2**62)
    M = len(vox["voxel_coords"])
    F = 0 if features is None else features.shape[1]
    feats = None if features is None else _f32(features)
    labs = None if classes is None else np.ascontiguousarray(classes, np.int32).reshape(-1)
    op = np.empty((M, 3), np.float32)
    of = np.empty((M, F), np.float32) if F else None
    ol = np.empty((M,), np.int32) if labs is not None else None
    rc = lib().oracle_voxel_reduce(
        _p(points, ctypes.c_float), ctypes.c_int(3), _p(feats, ctypes.c_float) if F else None, ctypes.c_int(F),
        _p(labs, ctypes.c_int32) if labs is not None else None, _p(vox["voxel_point_row_splits"], ctypes.c_int64),
        _p(vox["voxel_point_indices"], ctypes.c_int64), ctypes.c_int64(M), ctypes.c_int(0), ctypes.c_int(0),
        _p(op, ctypes.c_float), _p(of, ctypes.c_float) if F else None, _p(ol, ctypes.c_int32) if ol is not None else None)
    assert rc == 0
    out = [op, np.diff(vox["voxel_batch_splits"]).astype(np.int32)]
    if F:
        out.append(of)
    if ol is not None:
        out.append(ol)
    return tuple(out)


def np_subsample_batch(points, batches_len, features=None, classes=None, sampleDl=0.1, max_p=0):
    """numpy restatement of c_subsample_batch (independent code path: np_voxelize + python loops)."""
    points = _f32(points)
    rs = np.concatenate([[0], np.cumsum(np.asarray(batches_len, np.int64))]).astype(np.int64)
    origin, mx = subsample_range(points, sampleDl)
    vox = np_voxelize(points, rs, [sampleDl] * 3, origin, mx, 2**62, max_p if max_p > 0 else 2**62)
    vrs, pidx = vox["voxel_point_row_splits"], vox["voxel_point_indices"]
    M = len(vox["voxel_coords"])

    def mean(src):
        out = np.empty((M, src.shape[1]), np.float32)
        for v in range(M):
            acc = np.zeros(src.shape[1], np.float32)
            for j in pidx[vrs[v]:vrs[v + 1]]:
                acc = (acc + src[j]).astype(np.float32)
            out[v] = (acc / np.float32(vrs[v + 1] - vrs[v])).astype(np.float32)
        return out
    out = [mean(points), np.diff(vox["voxel_batch_splits"]).astype(np.int32)]
    if features is not None:
        out.append(mean(_f32(features)))
    if classes is not None:
        labs = np.asarray(classes, np.int32).reshape(-1)
        ol = np.empty(M, np.int32)
        for v in range(M):
            vals, cnt = np.unique(labs[pidx[vrs[v]:vrs[v + 1]]], return_counts=True)
            ol[v] = vals[np.argmax(cnt)]          # np.unique sorts: first maximum = smallest label
        out.append(ol)
    return tuple(out)


# ----------------------------------------------------------------------------
# rotated IoU / NMS (contract: ops_ref.c, "rotated IoU / NMS")
# ----------------------------------------------------------------------------
def c_iou_matrix(a, b, mode):
    a, b = _f32(a), _f32(b)
    out = np.zeros((len(a), len(b)), np.float32)
    if len(a) and len(b):
        assert lib().oracle_iou_matrix(_p(a, ctypes.c_float), ctypes.c_int64(len(a)), _p(b, ctypes.c_float),
                                       ctypes.c_int64(len(b)), ctypes.c_int(mode), _p(out, ctypes.c_float)) == 0
    return out


def c_nms(boxes, scores, thr):
    """-> (keep int64 [K], min |IoU - thr| over the decisive comparisons)."""
    boxes, scores = _f32(boxes), _f32(scores)
    keep = np.empty(max(len(boxes), 1), np.int64)
    gap = ctypes.c_double()
    L = lib()
    L.oracle_nms.restype = ctypes.c_int64
    k = L.oracle_nms(_p(boxes, ctypes.c_float), _p(scores, ctypes.c_float), ctypes.c_int64(len(boxes)),
                     ctypes.c_float(thr), _p(keep, ctypes.c_int64), ctypes.byref(gap))
    return keep[:k].copy(), gap.value


def np_rbox_area_mc(a, b, samples=400000, seed=0):
    """Monte-Carlo estimate of the intersection area of two (cx, cy, w, h, r) boxes: an independent check."""
    rng = np.random.default_rng(seed)
    r = max(a[2], a[3], b[2], b[3])
    lo = np.minimum(a[:2], b[:2]) - r
    hi = np.maximum(a[:2], b[:2]) + r
    p = rng.random((samples, 2)) * (hi - lo) + lo

    def inside(bx):
        c, s = np.cos(bx[4]), np.sin(bx[4])
        d = p - bx[:2]
        u, v = d[:, 0] * c + d[:, 1] * s, -d[:, 0] * s + d[:, 1] * c
        return (np.abs(u) <= bx[2] / 2) & (np.abs(v) <= bx[3] / 2)
    return float(np.mean(inside(a) & inside(b)) * np.prod(hi - lo))


# ----------------------------------------------------------------------------
# sparse convolution / segment sums (contract: ops_ref.c)
# ----------------------------------------------------------------------------
def c_sparse_conv(feat, in_pos, out_pos, voxel_size, offset, kernel, bias=None, normalize=False, transpose=False):
    feat, in_pos, out_pos, kernel = _f32(feat), _f32(in_pos), _f32(out_pos), _f32(kernel)
    ks = np.ascontiguousarray(kernel.shape[:3], np.int32)
    cin, cout = kernel.shape[3], kernel.shape[4]
    off = _f32(offset).reshape(3)
    out = np.zeros((len(out_pos), cout), np.float32)
    b = None if bias is None else _f32(bias)
    rc = lib().oracle_sparse_conv(_p(feat, ctypes.c_float), _p(in_pos, ctypes.c_float), ctypes.c_int64(len(in_pos)),
                                  _p(out_pos, ctypes.c_float), ctypes.c_int64(len(out_pos)), ctypes.c_float(voxel_size),
                                  _p(off, ctypes.c_float), _p(ks, ctypes.c_int), ctypes.c_int(int(transpose)),
                                  _p(kernel, ctypes.c_float), ctypes.c_int(cin), ctypes.c_int(cout),
                                  _p(b, ctypes.c_float) if b is not None else None, ctypes.c_int(int(normalize)),
                                  _p(out, ctypes.c_float))
    assert rc == 0
    return out


def c_reduce_subarrays_sum(values, row_splits):
    values, rs = _f32(values), np.ascontiguousarray(row_splits, np.int64)
    out = np.zeros(len(rs) - 1, np.float32)
    assert lib().oracle_reduce_subarrays_sum(_p(values, ctypes.c_float), _p(rs, ctypes.c_int64),
                                             ctypes.c_int64(len(rs) - 1), _p(out, ctypes.c_float)) == 0
    return out


def c_continuous_conv(filters, out_pos, extents, offset, inp_pos, feat, inp_imp, nbr, nbr_imp, splits,
                      align_corners, mapping, normalize, interp):
    """mapping / interp are the integer codes of cconv.cu."""
    filters, out_pos, inp_pos, feat = _f32(filters), _f32(out_pos), _f32(inp_pos), _f32(feat)
    ext = _f32(np.asarray(extents).reshape(-1))
    sz, sy, sx, cin, cout = filters.shape
    nbr = np.ascontiguousarray(nbr, np.int64)
    splits = np.ascontiguousarray(splits, np.int64)
    out = np.zeros((len(out_pos), cout), np.float32)
    ii = None if inp_imp is None else _f32(inp_imp)
    ni = None if nbr_imp is None else _f32(nbr_imp)
    off = _f32(offset).reshape(3)
    rc = lib().oracle_continuous_conv(
        _p(filters, ctypes.c_float), sx, sy, sz, cin, cout, _p(out_pos, ctypes.c_float), ctypes.c_int64(len(out_pos)),
        _p(ext, ctypes.c_float), int(len(ext) > 1), _p(off, ctypes.c_float), _p(inp_pos, ctypes.c_float),
        _p(feat, ctypes.c_float), _p(ii, ctypes.c_float) if ii is not None else None, _p(nbr, ctypes.c_int64),
        _p(ni, ctypes.c_float) if ni is not None else None, _p(splits, ctypes.c_int64), int(align_corners), int(mapping),
        int(normalize), int(interp), _p(out, ctypes.c_float))
    assert rc == 0
    return out
