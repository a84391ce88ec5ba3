"""Host-side mirror of ``open3d.ml.torch.ops`` / ``open3d.ml.torch.layers`` /
``open3d.core.nns`` for the operators on the hot path (SURVEY.md section 2.2),
backed by the sm_90a kernels of libo3dml_b200.so.

Same names, argument meaning, result field names and error behaviour
(RuntimeError) as the interface the reference's models call:

    voxelize          ml3d/torch/models/point_pillars.py:354-357
    ragged_to_dense   point_pillars.py:364-366, kpconv.py:2030-2032
    knn_search        ml3d/torch/models/point_transformer.py:724-734
    FixedRadiusSearch ml3d/torch/models/kpconv.py:2021-2026
    radius_search / RadiusSearch, and the metric / ignore_query_point / index_dtype options of the
                      searches (no call site; contract in DESIGN.md section 2)
    NearestNeighborSearch  ml3d/datasets/utils/dataprocessing.py:99-103

Inputs may live on the CPU (the reference's dataloaders call these ops with
numpy-backed tensors): they are copied to the current CUDA device, the kernels
run there, and the results come back on the input's device.  There is no CPU
implementation.
"""
import collections

import numpy as np
import torch

from . import _lib as L
from . import layers

VoxelizeResult = collections.namedtuple(
    "VoxelizeResult",
    "voxel_coords voxel_point_indices voxel_point_row_splits voxel_batch_splits")
KnnResult = collections.namedtuple("KnnSearchResult",
                                   "neighbors_index neighbors_row_splits neighbors_distance")
RadiusResult = collections.namedtuple("FixedRadiusSearchResult",
                                      "neighbors_index neighbors_row_splits neighbors_distance")

INT64_MAX = 2**63 - 1


def _dev(t):
    L.require_cuda()
    return t if t.is_cuda else t.cuda(non_blocking=True)


def _back(out, dev):
    """An op's result -- a tensor, None or a namedtuple of them -- handed back on `dev`, the device of the caller's
    input: results computed on the GPU are copied to the host for a host caller; host tensors stay as they are."""
    def back(t):
        return t if t is None or not t.is_cuda else t.to(dev)
    return out._make(map(back, out)) if isinstance(out, tuple) else back(out)


def _host3(x, what):
    a = np.ascontiguousarray(torch.as_tensor(x).detach().cpu().numpy(), dtype=np.float32).reshape(-1)
    if a.size != 3:
        raise RuntimeError("%s must have 3 elements, got %d" % (what, a.size))
    return a


def _check_points(points, name="points"):
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError("%s must have shape [N,3], got %s" % (name, tuple(points.shape)))
    if points.dtype != torch.float32:
        raise RuntimeError("%s must be float32" % name)


def _row_splits(row_splits):
    if row_splits.dtype != torch.int64:
        raise RuntimeError("row_splits must be int64")
    return _dev(row_splits).contiguous()


def _splits(row_splits, n, device):
    """_row_splits, or one batch item of n rows when row_splits is None."""
    if row_splits is None:
        return torch.tensor([0, n], dtype=torch.int64, device=device)
    return _row_splits(row_splits)


def voxelize_raw(points, row_splits, voxel_size, points_range_min, points_range_max,
                 max_points_per_voxel, max_voxels, want_batch_id=False):
    """Sync-free form: worst-case sized CUDA outputs + a device counter.
    points may be a strided [N,3] view of an [N,C] tensor (last-dim stride 1)."""
    _check_points(points)
    points = _dev(points)
    if points.stride(1) != 1:
        points = points.contiguous()
    n = points.shape[0]
    dev = points.device
    rs = _splits(row_splits, n, dev)
    batch = rs.numel() - 1
    vs, rmin, rmax = (_host3(voxel_size, "voxel_size"), _host3(points_range_min, "points_range_min"),
                      _host3(points_range_max, "points_range_max"))
    coords = torch.empty((n, 3), dtype=torch.int32, device=dev)
    pidx = torch.empty((n,), dtype=torch.int64, device=dev)
    vrs = torch.empty((n + 1,), dtype=torch.int64, device=dev)
    bsp = torch.empty((batch + 1,), dtype=torch.int64, device=dev)
    bid = torch.empty((n,), dtype=torch.int32, device=dev) if want_batch_id else None
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    ws = L.workspace(L.lib().o3dml_voxelize_workspace_bytes(n, batch), dev)
    L.check(L.lib().o3dml_voxelize(
        L.ptr(points), n, points.stride(0), L.ptr(rs), batch, vs.ctypes.data, rmin.ctypes.data,
        rmax.ctypes.data, int(min(max_points_per_voxel, INT64_MAX)), int(min(max_voxels, INT64_MAX)),
        L.ptr(coords), L.ptr(pidx), L.ptr(vrs), L.ptr(bsp), L.ptr(bid), L.ptr(counts), L.ptr(ws),
        ws.numel(), L.stream()))
    return coords, pidx, vrs, bsp, bid, counts


def voxelize(points, row_splits, voxel_size, points_range_min, points_range_max,
             max_points_per_voxel=INT64_MAX, max_voxels=INT64_MAX):
    """open3d.ml.torch.ops.voxelize -- one device->host read (the voxel count)."""
    coords, pidx, vrs, bsp, _, counts = voxelize_raw(points, row_splits, voxel_size,
                                                     points_range_min, points_range_max,
                                                     max_points_per_voxel, max_voxels)
    m, kept = (int(v) for v in counts.tolist())
    return _back(VoxelizeResult(coords[:m], pidx[:kept], vrs[:m + 1], bsp), points.device)


def ragged_to_dense(values, row_splits, out_col_size, default_value, _add=0):
    """open3d.ml.torch.ops.ragged_to_dense for integer / float32 values of shape [L] or [L, ...]."""
    v = _dev(values).contiguous()
    if v.element_size() not in (4, 8):
        raise RuntimeError("ragged_to_dense: 4- or 8-byte element types only")
    rs = _row_splits(row_splits)
    rows = rs.numel() - 1
    inner = 1
    for s in v.shape[1:]:
        inner *= s
    out = torch.empty((rows, int(out_col_size)) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
    fill = torch.as_tensor(default_value).reshape(-1)[:1].to(v.dtype)
    if v.dtype.is_floating_point:
        if _add != 0:
            raise RuntimeError("ragged_to_dense: add is for integer types")
        bits = int(fill.view(torch.int32 if v.element_size() == 4 else torch.int64).item())
    else:
        bits = int(fill.item())
    L.check(L.lib().o3dml_ragged_to_dense(L.ptr(v), v.element_size(), inner, L.ptr(rs), rows,
                                          int(out_col_size), bits, int(_add), L.ptr(out), L.stream()))
    return _back(out, values.device)


def knn_workspace_bytes(num_points, num_queries, batch):
    return L.lib().o3dml_knn_workspace_bytes(num_points, num_queries, batch)


def knn_search_raw(points, points_row_splits, queries, queries_row_splits, k, out_index, out_distance2=None,
                   workspace=None):
    """Sync-free form of knn_search: contiguous CUDA points / queries [N,3] with int64 row splits, dense outputs from
    the caller (out_index int32 or int64 [Nq, k], out_distance2 float32 [Nq, k] or None), and a uint8 workspace of
    at least knn_workspace_bytes, allocated here when none is given."""
    batch = points_row_splits.numel() - 1
    if workspace is None:
        workspace = L.workspace(knn_workspace_bytes(points.shape[0], queries.shape[0], batch), points.device)
    L.check(L.lib().o3dml_knn_search(L.ptr(points), points.shape[0], L.ptr(points_row_splits), L.ptr(queries),
                                     queries.shape[0], L.ptr(queries_row_splits), batch, int(k), L.ptr(out_index),
                                     L.is64(out_index), L.ptr(out_distance2), L.ptr(workspace), workspace.numel(),
                                     L.stream()))


_METRICS = {"L2": 0, "L1": 1, "Linf": 2}


def _metric(metric, name):
    if metric not in _METRICS:
        raise RuntimeError("%s: metric must be one of L1, L2, Linf (got %r)" % (name, metric))
    return _METRICS[metric]


def _index_dtype(index_dtype, name):
    if index_dtype not in (torch.int32, torch.int64):
        raise RuntimeError("%s: index_dtype must be torch.int32 or torch.int64" % name)
    return index_dtype


def _search_args(name, points, queries, points_row_splits, queries_row_splits, index_dtype, metric):
    """The checks every search makes, in order, and its inputs on the device: (metric code, points, queries, their
    row splits, batch size)."""
    m = _metric(metric, name)
    _index_dtype(index_dtype, name)
    _check_points(points), _check_points(queries, "queries")
    p, q = _dev(points).contiguous(), _dev(queries).contiguous()
    ps, qs = _splits(points_row_splits, p.shape[0], p.device), _splits(queries_row_splits, q.shape[0], p.device)
    batch = ps.numel() - 1
    if qs.numel() - 1 != batch:
        raise RuntimeError("%s: row splits disagree on the batch size" % name)
    return m, p, q, ps, qs, batch


def knn_search(points, queries, k, points_row_splits=None, queries_row_splits=None,
               index_dtype=torch.int32, metric="L2", ignore_query_point=False,
               return_distances=False, allow_short=False):
    """open3d.ml.torch.ops.knn_search.  Rows ascend by (distance, index) in `metric` (L1, L2, Linf); L2 distances are
    squared, as upstream returns them.  Dense [Nq * k] rows with row splits 0, k, 2k, ...; with ignore_query_point
    (points equal to the query are skipped) a row may hold fewer than k neighbours, and the rows are ragged (one
    device->host read of their total).  NaN distances are never ranked and +inf ones rank last, so a row that finds
    fewer than k rankable points (NaN coordinates) is padded with index -1 and distance +inf: dense rows in place,
    ragged rows by their length."""
    m, p, q, ps, qs, batch = _search_args("knn_search", points, queries, points_row_splits, queries_row_splits,
                                          index_dtype, metric)
    dev = p.device
    k = int(k)
    # upstream returns ragged (shorter) rows when a batch item holds fewer than k points; this op returns dense
    # [Nq, k] rows, so refuse instead of handing out -1 padded indices that a caller would gather with
    short = int((ps[1:] - ps[:-1]).min()) if batch > 0 and q.shape[0] > 0 and not allow_short else k
    if short < k:      # allow_short=True keeps the C-ABI behaviour: -1 / +inf padded dense rows
        raise RuntimeError("knn_search: a batch item has %d points, fewer than k = %d (ragged results are not "
                           "implemented)" % (short, k))
    nq = q.shape[0]
    if m == 0 and not ignore_query_point:
        idx = torch.empty((nq, k), dtype=index_dtype, device=dev)
        d2 = torch.empty((nq, k), dtype=torch.float32, device=dev) if return_distances else None
        knn_search_raw(p, ps, q, qs, k, idx, d2)
        rs = torch.arange(0, (nq + 1) * k, k, dtype=torch.int64, device=dev)
    else:
        ig = 1 if ignore_query_point else 0
        idx = torch.empty((nq * k,), dtype=index_dtype, device=dev)
        d2 = torch.empty((nq * k,), dtype=torch.float32, device=dev) if return_distances else None
        rs = torch.arange(0, (nq + 1) * k, k, dtype=torch.int64, device=dev) if not ig else \
            torch.empty((nq + 1,), dtype=torch.int64, device=dev)
        total = torch.zeros((1,), dtype=torch.int64, device=dev)
        ws = L.workspace(L.lib().o3dml_knn_search_metric_workspace_bytes(p.shape[0], nq, batch, k, ig), dev)
        L.check(L.lib().o3dml_knn_search_metric(L.ptr(p), p.shape[0], L.ptr(ps), L.ptr(q), nq, L.ptr(qs), batch, k, m,
                                                ig, L.ptr(idx), L.is64(idx), L.ptr(d2), L.ptr(rs), L.ptr(total),
                                                L.ptr(ws), ws.numel(), L.stream()))
        if ig:
            t = int(total.item())
            idx, d2 = idx[:t], (d2[:t] if d2 is not None else None)
    out = KnnResult(idx.reshape(-1), rs,
                    d2.reshape(-1) if d2 is not None else torch.empty(0, device=dev))
    return _back(out, points.device)


def _radius_search(name, points, queries, radius, radii, points_row_splits, queries_row_splits, index_dtype, metric,
                   ignore_query_point, return_distances, normalize_distances):
    """Two-phase radius search (count, one device->host read of the total, fill) with one radius (radii None) or
    one per query."""
    m, p, q, ps, qs, batch = _search_args(name, points, queries, points_row_splits, queries_row_splits, index_dtype,
                                          metric)
    dev = p.device
    nq = q.shape[0]
    if radii is not None:
        radii = _dev(torch.as_tensor(radii)).reshape(-1).contiguous()
        if radii.dtype != torch.float32 or radii.numel() != nq:
            raise RuntimeError("%s: radii must be float32 with one radius per query (%d)" % (name, nq))
    ig, norm = 1 if ignore_query_point else 0, 1 if normalize_distances else 0
    nrs = torch.empty((nq + 1,), dtype=torch.int64, device=dev)
    total = torch.zeros((1,), dtype=torch.int64, device=dev)
    ws = L.workspace(L.lib().o3dml_radius_workspace_bytes(p.shape[0], nq, batch), dev)
    L.check(L.lib().o3dml_radius_search_count(L.ptr(p), p.shape[0], L.ptr(ps), L.ptr(q), nq, L.ptr(qs), batch,
                                              float(radius), L.ptr(radii), m, ig, L.ptr(nrs), L.ptr(total), L.ptr(ws),
                                              ws.numel(), L.stream()))
    t = int(total.item())
    idx = torch.empty((t,), dtype=index_dtype, device=dev)
    d = torch.empty((t,), dtype=torch.float32, device=dev)
    if t:      # with no neighbour at all there is nothing to fill (and the empty outputs have no address)
        L.check(L.lib().o3dml_radius_search_fill(L.ptr(q), p.shape[0], nq, L.ptr(qs), batch, float(radius),
                                                 L.ptr(radii), m, ig, norm, L.ptr(nrs), L.ptr(idx), L.is64(idx),
                                                 L.ptr(d), L.ptr(ws), ws.numel(), L.stream()))
    return _back(RadiusResult(idx, nrs, d if return_distances else torch.empty(0, device=dev)), points.device)


def fixed_radius_search(points, queries, radius, points_row_splits=None, queries_row_splits=None,
                        return_distances=True, index_dtype=torch.int32, metric="L2", ignore_query_point=False):
    """open3d.ml.torch.ops.fixed_radius_search: the points within `radius` (> 0) of each query in `metric` (L1, L2,
    Linf; L2 distances squared), rows by (distance, index); ignore_query_point skips points equal to the query.  Two
    phases (count, one device->host read of the total, fill)."""
    return _radius_search("fixed_radius_search", points, queries, radius, None, points_row_splits, queries_row_splits,
                          index_dtype, metric, ignore_query_point, return_distances, False)


def radius_search(points, queries, radii, points_row_splits=None, queries_row_splits=None, index_dtype=torch.int32,
                  metric="L2", ignore_query_point=False, return_distances=False, normalize_distances=False):
    """open3d.ml.torch.ops.radius_search: fixed_radius_search with one radius per query, radii float32 [Nq].  A
    negative, NaN or infinite radius gives an empty row; r = 0 keeps the points equal to the query.
    normalize_distances returns distance / (r * r) for L2 and distance / r otherwise (NaN for r = 0)."""
    return _radius_search("radius_search", points, queries, 0.0, radii, points_row_splits, queries_row_splits,
                          index_dtype, metric, ignore_query_point, return_distances, normalize_distances)


class FixedRadiusSearch(torch.nn.Module):
    """open3d.ml.torch.layers.FixedRadiusSearch (kpconv.py:2021-2026).  A prebuilt hash_table is accepted and not
    used: the search builds its own grid."""

    def __init__(self, metric="L2", ignore_query_point=False, return_distances=False,
                 max_hash_table_size=32 * 2**20, index_dtype=torch.int32, **kwargs):
        super().__init__()
        _metric(metric, "FixedRadiusSearch")
        self.kw = dict(metric=metric, ignore_query_point=ignore_query_point,
                       return_distances=return_distances, index_dtype=_index_dtype(index_dtype, "FixedRadiusSearch"))

    def forward(self, points, queries, radius, points_row_splits=None, queries_row_splits=None,
                hash_table_size_factor=1 / 64, hash_table=None):
        return fixed_radius_search(points, queries, radius, points_row_splits, queries_row_splits, **self.kw)


class RadiusSearch(torch.nn.Module):
    """open3d.ml.torch.layers.RadiusSearch: radius_search with one radius per query."""

    def __init__(self, metric="L2", ignore_query_point=False, return_distances=False, normalize_distances=False,
                 index_dtype=torch.int32, **kwargs):
        super().__init__()
        _metric(metric, "RadiusSearch")
        self.kw = dict(metric=metric, ignore_query_point=ignore_query_point, return_distances=return_distances,
                       normalize_distances=normalize_distances,
                       index_dtype=_index_dtype(index_dtype, "RadiusSearch"))

    def forward(self, points, queries, radii, points_row_splits=None, queries_row_splits=None):
        return radius_search(points, queries, radii, points_row_splits, queries_row_splits, **self.kw)


class KNNSearch(torch.nn.Module):
    """open3d.ml.torch.layers.KNNSearch."""

    def __init__(self, metric="L2", ignore_query_point=False, return_distances=False,
                 index_dtype=torch.int32, **kwargs):
        super().__init__()
        _metric(metric, "KNNSearch")
        self.kw = dict(metric=metric, ignore_query_point=ignore_query_point,
                       return_distances=return_distances, index_dtype=_index_dtype(index_dtype, "KNNSearch"))

    def forward(self, points, queries, k, points_row_splits=None, queries_row_splits=None):
        return knn_search(points, queries, k, points_row_splits, queries_row_splits, **self.kw)


class _O3CTensor:
    """The sliver of open3d.core.Tensor that dataprocessing.py:99-103 touches."""

    def __init__(self, t):
        self.t = t

    @staticmethod
    def from_numpy(a):
        return _O3CTensor(torch.from_numpy(np.ascontiguousarray(a)))

    def numpy(self):
        return self.t.cpu().numpy()


class NearestNeighborSearch:
    """open3d.core.nns.NearestNeighborSearch: knn_index(); knn_search(queries, k) -> (idx int64, d2)."""

    def __init__(self, dataset_points, index_dtype=None):
        t = dataset_points.t if isinstance(dataset_points, _O3CTensor) else torch.as_tensor(dataset_points)
        self.points = _dev(t.to(torch.float32)).contiguous()

    def knn_index(self):
        return True

    def knn_search(self, query_points, knn):
        q = query_points.t if isinstance(query_points, _O3CTensor) else torch.as_tensor(query_points)
        q = _dev(q.to(torch.float32)).contiguous()
        r = knn_search(self.points, q, knn, index_dtype=torch.int64, return_distances=True)
        n = q.shape[0]
        return (_O3CTensor(r.neighbors_index.reshape(n, knn)),
                _O3CTensor(r.neighbors_distance.reshape(n, knn)))


# ------------------------------------------------------------------ grid subsampling
def voxel_reduce(points, features, labels, vrs, pidx, counts=None, num_voxels=None,
                 position_mode=0, feature_mode=0, want_points=True):
    """Per-voxel mean / max / first over CSR voxel lists (o3dml_voxel_reduce).  All CUDA tensors."""
    m = int(num_voxels if num_voxels is not None else vrs.numel() - 1)
    dev = points.device
    F = 0 if features is None else features.shape[1]
    op = torch.empty((m, 3), dtype=torch.float32, device=dev) if want_points else None
    of = torch.empty((m, F), dtype=torch.float32, device=dev) if F else None
    ol = torch.empty((m,), dtype=torch.int32, device=dev) if labels is not None else None
    L.check(L.lib().o3dml_voxel_reduce(
        L.ptr(points), points.stride(0), L.ptr(features), F, features.stride(0) if F else 0, L.ptr(labels),
        L.ptr(vrs), L.ptr(pidx), L.ptr(counts), m, int(position_mode), int(feature_mode), L.ptr(op), L.ptr(of),
        L.ptr(ol), L.stream()))
    return op, of, ol


def _subsample_range(pts, dl):
    """Grid origin = the largest float32 <= floor(min / dl) * dl, upper bound = max: ONE device->host read.

    The origin is worked out in float64 with dl at its float32 value.  k * dl is then exact (a 24-bit significand
    times an integer, exact while |min / dl| < 2^29), so the one rounding of min / dl is corrected by a comparison, and the origin is rounded down
    to float32: origin <= min on every axis, so voxelize's `origin <= p` test keeps the cloud's minimum.  A float32
    product rounded to nearest can land above min (min = -58.2, dl = 0.04 gives -58.199997) and drop that point."""
    mm = torch.stack([pts.amin(0), pts.amax(0)]).cpu().numpy().astype(np.float32)
    if not np.isfinite(mm).all():
        raise RuntimeError("subsample: the points must be finite (min %s, max %s)" % (mm[0], mm[1]))
    mn, d = mm[0].astype(np.float64), np.float64(np.float32(dl))
    k = np.floor(mn / d)
    k -= k * d > mn
    o64 = k * d
    origin = o64.astype(np.float32)
    origin = np.where(origin > o64, np.nextafter(origin, np.float32(-np.inf)), origin).astype(np.float32)
    return origin, mm[1]


def subsample_batch_cuda(points, row_splits, features=None, classes=None, sampleDl=0.1, max_p=0):
    """Grid subsampling of a stacked batch on the device: CUDA tensors in, CUDA tensors out.
    Returns (s_points [M,3], s_row_splits int64 [B+1], s_features or None, s_labels or None)."""
    _check_points(points)
    pts = _dev(points).contiguous()
    if pts.shape[0] == 0:
        raise RuntimeError("subsample: empty point cloud")
    rs = _splits(row_splits, pts.shape[0], pts.device)
    origin, mx = _subsample_range(pts, sampleDl)
    dl = float(sampleDl)
    coords, pidx, vrs, bsp, _, counts = voxelize_raw(pts, rs, [dl, dl, dl], origin, mx, INT64_MAX,
                                                     int(max_p) if max_p and max_p > 0 else INT64_MAX)
    m = int(counts[0].item())
    feats = None if features is None else _dev(features).to(torch.float32).contiguous()
    labs = None if classes is None else _dev(classes).to(torch.int32).contiguous().view(-1)
    if feats is not None and feats.dim() == 1:
        feats = feats.view(-1, 1)
    op, of, ol = voxel_reduce(pts, feats, labs, vrs, pidx, counts, m)
    return op, bsp, of, ol


def subsample_batch(points, batches_len, features=None, classes=None, sampleDl=0.1, method="barycenter",
                    max_p=0, verbose=0):
    """open3d.ml.contrib.subsample_batch (ml3d/torch/models/kpconv.py:2096-2164): numpy in, numpy out.
    Returns (s_points, s_len[, s_features][, s_labels]) exactly like the call sites unpack it."""
    if method != "barycenter":
        raise RuntimeError("subsample_batch: only method='barycenter' is implemented")
    pts = torch.as_tensor(np.ascontiguousarray(points, dtype=np.float32))
    lens = np.asarray(batches_len, dtype=np.int64).reshape(-1)
    rs = torch.as_tensor(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    f = None if features is None else torch.as_tensor(np.ascontiguousarray(features, dtype=np.float32))
    c = None if classes is None else torch.as_tensor(np.ascontiguousarray(classes).astype(np.int32))
    op, bsp, of, ol = subsample_batch_cuda(pts, rs, f, c, sampleDl, max_p)
    out = [op.cpu().numpy(), np.diff(bsp.cpu().numpy()).astype(np.int32)]
    if of is not None:
        out.append(of.cpu().numpy())
    if ol is not None:
        lab = ol.cpu().numpy()
        out.append(lab.astype(np.asarray(classes).dtype, copy=False))
    return tuple(out)


def subsample(points, features=None, classes=None, sampleDl=0.1, verbose=0):
    """open3d.ml.contrib.subsample (ml3d/datasets/utils/dataprocessing.py:14-49): one cloud."""
    r = subsample_batch(points, [len(points)], features, classes, sampleDl)
    out = (r[0],) + tuple(r[2:])
    return out[0] if len(out) == 1 else out


# ------------------------------------------------------------------ detection post-processing
def nms(boxes, scores, nms_overlap_thresh):
    """open3d.ml.torch.ops.nms (ml3d/torch/utils/objdet_helper.py:346): boxes [N,5] = (x0, y0, x1, y1, r),
    scores [N] -> int64 indices of the kept boxes by descending score.  One device->host read (the count)."""
    if boxes.dim() != 2 or boxes.shape[1] != 5:
        raise RuntimeError("nms: boxes must have shape [N,5], got %s" % (tuple(boxes.shape),))
    if scores.dim() != 1 or scores.shape[0] != boxes.shape[0]:
        raise RuntimeError("nms: scores must have shape [N]")
    b = _dev(boxes).to(torch.float32).contiguous()
    s = _dev(scores).to(torch.float32).contiguous()
    n = b.shape[0]
    keep = torch.empty((n,), dtype=torch.int64, device=b.device)
    cnt = torch.zeros((1,), dtype=torch.int64, device=b.device)
    ws = L.workspace(L.lib().o3dml_nms_workspace_bytes(n), b.device)
    L.check(L.lib().o3dml_nms(L.ptr(b), L.ptr(s), n, float(nms_overlap_thresh), L.ptr(keep), L.ptr(cnt), L.ptr(ws),
                              ws.numel(), L.stream()))
    return _back(keep[:int(cnt.item())], boxes.device)


def _iou(a, b, mode, width):
    a_np, b_np = isinstance(a, np.ndarray), isinstance(b, np.ndarray)
    ta = torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)) if a_np else a
    tb = torch.as_tensor(np.ascontiguousarray(b, dtype=np.float32)) if b_np else b
    if ta.dim() != 2 or tb.dim() != 2 or ta.shape[1] != width or tb.shape[1] != width:
        raise RuntimeError("iou: boxes must have shape [N,%d]" % width)
    ta, tb = _dev(ta).to(torch.float32).contiguous(), _dev(tb).to(torch.float32).contiguous()
    out = torch.zeros((ta.shape[0], tb.shape[0]), dtype=torch.float32, device=ta.device)
    L.check(L.lib().o3dml_iou_matrix(L.ptr(ta), ta.shape[0], L.ptr(tb), tb.shape[0], mode, L.ptr(out), L.stream()))
    return out.cpu().numpy() if a_np else out


def iou_bev(boxes_a, boxes_b):
    """open3d.ml.contrib.iou_bev_{cpu,cuda} (ml3d/metrics/mAP.py:85): [N,5] x [M,5] (x, y, w, h, r) -> [N,M]."""
    return _iou(boxes_a, boxes_b, 0, 5)


def iou_3d(boxes_a, boxes_b):
    """open3d.ml.contrib.iou_3d_{cpu,cuda} (ml3d/metrics/mAP.py:88): [N,7] x [M,7] (x, y, z, w, h, l, ry)."""
    return _iou(boxes_a, boxes_b, 1, 7)


# ------------------------------------------------------------------ SparseConvUnet / op-surface ops (f3, f4)
def reduce_subarrays_sum(values, row_splits):
    """open3d.ml.torch.ops.reduce_subarrays_sum (ml3d/torch/models/sparseconvnet.py:318-324)."""
    if values.dim() != 1:
        raise RuntimeError("reduce_subarrays_sum: values must be 1-D")
    rs = _row_splits(row_splits)
    v = _dev(values).to(torch.float32).contiguous()
    rows = rs.numel() - 1
    out = torch.empty((max(rows, 0),), dtype=torch.float32, device=v.device)
    L.check(L.lib().o3dml_reduce_subarrays_sum(L.ptr(v), L.ptr(rs), rows, L.ptr(out), L.stream()))
    return _back(out.to(values.dtype), values.device)


VoxelPoolingResult = collections.namedtuple("VoxelPoolingResult", "pooled_positions pooled_features")
_POOL_MODES = {"average": 0, "max": 1, "nearest_neighbor": 2, "center": 3}


def voxel_pooling(positions, features, voxel_size, position_fn="average", feature_fn="average", debug=False):
    """open3d.ml.torch.ops.voxel_pooling (north-star op surface; no call site in the reference): one output
    point per occupied voxel of the grid anchored at the origin (voxel index = floor(p / voxel_size)).
    position_fn in {average, nearest_neighbor, center}, feature_fn in {average, max, nearest_neighbor};
    voxels come out in ascending (x + ex * (y + ey * z)) order.  'nearest_neighbor' takes the point closest to the
    voxel centre (ties: lowest index)."""
    if position_fn not in ("average", "nearest_neighbor", "center") or feature_fn not in ("average", "max", "nearest_neighbor"):
        raise RuntimeError("voxel_pooling: unknown position_fn / feature_fn")
    _check_points(positions, "positions")
    pts = _dev(positions).contiguous()
    feats = _dev(features).to(torch.float32).contiguous()
    if feats.dim() != 2 or feats.shape[0] != pts.shape[0]:
        raise RuntimeError("voxel_pooling: features must have shape [N, C]")
    if pts.shape[0] == 0:
        return _back(VoxelPoolingResult(pts.new_zeros((0, 3)), feats.new_zeros((0, feats.shape[1]))), positions.device)
    vs = float(voxel_size)
    origin, mx = _subsample_range(pts, vs)
    coords, pidx, vrs, bsp, _, counts = voxelize_raw(pts, None, [vs, vs, vs], origin, mx, INT64_MAX, INT64_MAX)
    m = int(counts[0].item())
    if "nearest_neighbor" in (position_fn, feature_fn):
        # reorder every voxel's point list so that its first entry is the point nearest to the voxel centre
        centre = (coords[:m].to(torch.float32) + 0.5) * vs + torch.from_numpy(origin).to(pts.device)
        vid = torch.repeat_interleave(torch.arange(m, device=pts.device), (vrs[1:m + 1] - vrs[:m]))
        d2 = ((pts[pidx[:vid.numel()]] - centre[vid]) ** 2).sum(1)
        order = torch.argsort(d2, stable=True)
        order = order[torch.argsort(vid[order], stable=True)]
        pidx = pidx.clone()
        pidx[:vid.numel()] = pidx[:vid.numel()][order]
    pm = {"average": 0, "nearest_neighbor": 2, "center": 2}[position_fn]
    fm = {"average": 0, "max": 1, "nearest_neighbor": 2}[feature_fn]
    op, of, _ = voxel_reduce(pts, feats, None, vrs, pidx, counts, m, position_mode=pm, feature_mode=fm)
    if position_fn == "center":
        op = (coords[:m].to(torch.float32) + 0.5) * vs + torch.from_numpy(origin).to(pts.device)
    return _back(VoxelPoolingResult(op, of), positions.device)


_CCONV_MAPPING = {"identity": 0, "ball_to_cube_radial": 1}
_CCONV_INTERP = {"nearest_neighbor": 0, "linear": 1, "linear_border": 2}


def _cconv_args(name, filters, out_positions, extents, offset, inp_positions, inp_features, neighbors_index,
                neighbors_row_splits, coordinate_mapping, interpolation, extents_per_inp):
    """The arguments continuous_conv and its transpose share, checked and on the device: (filters, out_positions,
    inp_positions, inp_features, extents, host offset, neighbors_index, neighbors_row_splits).  Positions are
    [N, 3] and inp_features [num_inp, Cin].  Per-point extents count the outputs, or the inputs when
    `extents_per_inp` (the transpose, which also refuses them with no input)."""
    if coordinate_mapping not in _CCONV_MAPPING:
        raise RuntimeError("%s: coordinate_mapping '%s' is not implemented (identity, ball_to_cube_radial)"
                           % (name, coordinate_mapping))
    if interpolation not in _CCONV_INTERP:
        raise RuntimeError("%s: unknown interpolation '%s'" % (name, interpolation))
    if filters.dim() != 5:
        raise RuntimeError("%s: filters must have shape [Sz, Sy, Sx, Cin, Cout]" % name)
    for what, t in (("out_positions", out_positions), ("inp_positions", inp_positions)):
        if t.dim() != 2 or t.shape[1] != 3:
            raise RuntimeError("%s: %s must have shape [N, 3], got %s" % (name, what, tuple(t.shape)))
    if inp_features.dim() != 2 or inp_features.shape[0] != inp_positions.shape[0] or \
            inp_features.shape[1] != filters.shape[3]:
        raise RuntimeError("%s: feature channels do not match the filter (inp_features must be [num_inp, Cin])"
                           % name)
    f = _dev(filters).to(torch.float32).contiguous()
    op, ip = _dev(out_positions).to(torch.float32).contiguous(), _dev(inp_positions).to(torch.float32).contiguous()
    feat = _dev(inp_features).to(torch.float32).contiguous()
    ext = _dev(torch.as_tensor(extents, dtype=torch.float32).reshape(-1)).contiguous()
    n, side = (ip.shape[0], "num_inp") if extents_per_inp else (op.shape[0], "num_out")
    if ext.numel() != 1 and (ext.numel() != n or extents_per_inp and n == 0):
        raise RuntimeError("%s: extents must have 1 or %s elements" % (name, side))
    off = _host3(offset, "offset")
    idx = _dev(neighbors_index).contiguous()
    if idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("%s: neighbors_index must be int32 or int64" % name)
    rs = _dev(neighbors_row_splits).to(torch.int64).contiguous()
    if rs.numel() != op.shape[0] + 1:
        raise RuntimeError("%s: neighbors_row_splits must have num_out + 1 elements" % name)
    return f, op, ip, feat, ext, off, idx, rs


def _cconv_opt(name, t, n, what):
    """An optional per-point or per-entry float argument of the continuous convolutions: None for None or an empty
    tensor ("all ones"), else float32 [n] on the device.  The kernels read it by index, so a short one is refused."""
    if t is None or t.numel() == 0:
        return None
    t = _dev(t).float().reshape(-1).contiguous()
    if t.numel() != n:
        raise RuntimeError("%s: %s must be empty or have %d elements" % (name, what, n))
    return t


def continuous_conv(filters, out_positions, extents, offset, inp_positions, inp_features, inp_importance,
                    neighbors_index, neighbors_importance, neighbors_row_splits, align_corners=False,
                    coordinate_mapping="ball_to_cube_radial", normalize=False, interpolation="linear",
                    max_temp_mem_MB=64):
    """open3d.ml.torch.ops.continuous_conv (raw op; contract in csrc/cconv.cu).  filters [Sz, Sy, Sx, Cin, Cout];
    empty importance tensors mean "all ones", others have num_inp (inp_importance) or one per neighbour entry
    (neighbors_importance) elements; extents [1] or [num_out]."""
    name = "continuous_conv"
    f, op, ip, feat, ext, off, idx, rs = _cconv_args(
        name, filters, out_positions, extents, offset, inp_positions, inp_features, neighbors_index,
        neighbors_row_splits, coordinate_mapping, interpolation, extents_per_inp=False)
    imp = _cconv_opt(name, inp_importance, ip.shape[0], "inp_importance")
    nimp = _cconv_opt(name, neighbors_importance, idx.numel(), "neighbors_importance")
    sz, sy, sx, cin, cout = f.shape
    out = torch.empty((op.shape[0], cout), dtype=torch.float32, device=f.device)
    L.check(L.lib().o3dml_continuous_conv(
        L.ptr(f), sx, sy, sz, cin, cout, L.ptr(op), op.shape[0], L.ptr(ext), 1 if ext.numel() > 1 else 0,
        off.ctypes.data, L.ptr(ip), L.ptr(feat), ip.shape[0], L.ptr(imp), L.ptr(idx),
        L.is64(idx), L.ptr(nimp), L.ptr(rs), 1 if align_corners else 0,
        _CCONV_MAPPING[coordinate_mapping], 1 if normalize else 0, _CCONV_INTERP[interpolation], L.ptr(out), L.stream()))
    return _back(out, inp_features.device)


InvertNeighborsListResult = collections.namedtuple(
    "InvertNeighborsListResult", "neighbors_index neighbors_row_splits neighbors_attributes")


def invert_neighbors_list(num_points, inp_neighbors_index, inp_neighbors_row_splits, inp_neighbors_attributes):
    """open3d.ml.torch.ops.invert_neighbors_list: num_inp rows of ids in [0, num_points) -> num_points rows of the
    input rows that contain each id, once per occurrence, by (input row, position in it): a stable sort by id.  Ids out
    of range are dropped (they follow the last row; neighbors_row_splits[-1] counts the entries kept).  The attributes
    ([E, ...], any dtype) are permuted the same way; an empty attributes tensor stays empty.  No host read."""
    idx = _dev(inp_neighbors_index).reshape(-1).contiguous()
    if idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("invert_neighbors_list: inp_neighbors_index must be int32 or int64")
    rs = _row_splits(inp_neighbors_row_splits)
    num_points, e, num_inp = int(num_points), idx.numel(), rs.numel() - 1
    if num_points < 0 or num_inp < 0:
        raise RuntimeError("invert_neighbors_list: num_points must be >= 0 and row_splits non-empty")
    attrs = inp_neighbors_attributes
    if attrs.numel() and attrs.shape[0] != e:
        raise RuntimeError("invert_neighbors_list: attributes must have one row per neighbour entry")
    dev = idx.device
    out_idx = torch.empty((e,), dtype=idx.dtype, device=dev)
    out_rs = torch.empty((num_points + 1,), dtype=torch.int64, device=dev)
    perm = torch.empty((e,), dtype=torch.int64, device=dev)
    ws = L.workspace(L.lib().o3dml_invert_neighbors_list_workspace_bytes(e), dev)
    L.check(L.lib().o3dml_invert_neighbors_list(num_points, L.ptr(idx), L.is64(idx), L.ptr(rs), num_inp, e,
                                                L.ptr(out_idx), L.ptr(out_rs), L.ptr(perm), L.ptr(ws), ws.numel(),
                                                L.stream()))
    out_attrs = _dev(attrs)[perm] if attrs.numel() else attrs
    return _back(InvertNeighborsListResult(out_idx, out_rs, out_attrs), inp_neighbors_index.device)


def trilinear_devoxelize_forward(resolution, is_training, coords, features):
    """open3d.ml.torch.ops.trilinear_devoxelize_forward (pvcnn.py:37): coords [B, 3, N] voxel coordinates in
    [0, r - 1], features [B, C, r, r, r] -> (outs [B, C, N], inds int32 [B, 8, N], wgts [B, 8, N]); the rule is in
    DESIGN.md section 2.  The kernel works on point rows and a channels-last grid, so the reference layout is
    permuted on the way in and out; the fused PVCNN forward keeps its own layout and skips that.  inds and wgts are
    written whether or not is_training is set.  No host read."""
    r = int(resolution)
    c, f = _dev(coords), _dev(features)
    if c.dim() != 3 or c.shape[1] != 3 or f.dim() != 5 or tuple(f.shape[2:]) != (r, r, r) or f.shape[0] != c.shape[0]:
        raise RuntimeError("trilinear_devoxelize_forward: coords [B, 3, N] and features [B, C, r, r, r] expected")
    if c.dtype != torch.float32 or f.dtype != torch.float32:
        raise RuntimeError("trilinear_devoxelize_forward: float32 inputs expected")
    B, _, N = c.shape
    C = f.shape[1]
    rows = c.permute(0, 2, 1).contiguous()
    grid = f.permute(0, 2, 3, 4, 1).contiguous()
    out = torch.empty((B, N, C), dtype=torch.float32, device=c.device)
    inds = torch.empty((B, 8, N), dtype=torch.int32, device=c.device)
    wgts = torch.empty((B, 8, N), dtype=torch.float32, device=c.device)
    L.check(L.lib().o3dml_trilinear_devoxelize(L.ptr(rows), B, N, r, L.ptr(grid), C, C, 0, L.ptr(out), C, L.ptr(inds),
                                               L.ptr(wgts), L.stream()))
    dev = coords.device
    return tuple(_back(t, dev) for t in (out.permute(0, 2, 1).contiguous(), inds, wgts))


def continuous_conv_transpose(filters, out_positions, out_importance, extents, offset, inp_positions, inp_features,
                              inp_neighbors_index, inp_neighbors_importance_sum, inp_neighbors_row_splits,
                              neighbors_index, neighbors_importance, neighbors_row_splits, align_corners=False,
                              coordinate_mapping="ball_to_cube_radial", normalize=False, interpolation="linear",
                              max_temp_mem_MB=64):
    """open3d.ml.torch.ops.continuous_conv_transpose (raw op; contract in csrc/cconv.cu), the adjoint of
    continuous_conv: filters [Sz, Sy, Sx, Cin, Cout] as there, inp_features [num_inp, Cin] -> [num_out, Cout].
    neighbors_* list the inputs of each output (invert_neighbors_list of the forward lists); extents [1] or
    [num_inp]; empty importance tensors mean "all ones".  Under normalize input i is scaled by
    1 / inp_neighbors_importance_sum[i], or by 1 / the length of its row of inp_neighbors_row_splits when that sum
    is empty.  inp_neighbors_index is taken for signature parity and not read.  No host read."""
    name = "continuous_conv_transpose"
    f, op, ip, feat, ext, off, idx, rs = _cconv_args(
        name, filters, out_positions, extents, offset, inp_positions, inp_features, neighbors_index,
        neighbors_row_splits, coordinate_mapping, interpolation, extents_per_inp=True)
    num_out, num_inp = op.shape[0], ip.shape[0]
    oimp = _cconv_opt(name, out_importance, num_out, "out_importance")
    isum = _cconv_opt(name, inp_neighbors_importance_sum, num_inp, "inp_neighbors_importance_sum")
    nimp = _cconv_opt(name, neighbors_importance, idx.numel(), "neighbors_importance")
    irs = None
    if inp_neighbors_row_splits is not None and inp_neighbors_row_splits.numel():
        irs = _dev(inp_neighbors_row_splits).to(torch.int64).contiguous()
        if irs.numel() != num_inp + 1:
            raise RuntimeError("%s: inp_neighbors_row_splits must have num_inp + 1 elements" % name)
    sz, sy, sx, cin, cout = f.shape
    out = torch.empty((num_out, cout), dtype=torch.float32, device=f.device)
    L.check(L.lib().o3dml_continuous_conv_transpose(
        L.ptr(f), sx, sy, sz, cin, cout, L.ptr(op), num_out, L.ptr(oimp), L.ptr(ext), 1 if ext.numel() > 1 else 0,
        off.ctypes.data, L.ptr(ip), L.ptr(feat), num_inp, L.ptr(isum), L.ptr(irs), L.ptr(idx), L.is64(idx),
        L.ptr(nimp), L.ptr(rs), 1 if align_corners else 0, _CCONV_MAPPING[coordinate_mapping], 1 if normalize else 0,
        _CCONV_INTERP[interpolation], L.ptr(out), L.stream()))
    return _back(out, inp_features.device)


def _sparse_filters(name, filters, feat):
    """filters [.., Cin, Cout] -> float32 CPU [cells, Cin, Cout], the leading dims flattened into the kernel index."""
    w = filters.detach().float().cpu()
    cin, cout = w.shape[-2], w.shape[-1]
    if feat.dim() != 2 or feat.shape[1] != cin:
        raise RuntimeError("%s: feature channels do not match the filter" % name)
    return w.reshape(-1, cin, cout)


def _sparse_importance(name, what, t, n, dev):
    """An importance argument: None for an empty tensor (all ones), else float32 [n] on `dev`."""
    if t is None or t.numel() == 0:
        return None
    t = _dev(t).to(dev, torch.float32).reshape(-1)
    if t.numel() != n:
        raise RuntimeError("%s: %s must be empty or have %d elements" % (name, what, n))
    return t


def _sparse_table(name, neighbors_index, neighbors_kernel_index, neighbors_row_splits, kc, num_in, dev,
                  entry_weight=None):
    """Ragged (index, kernel cell) lists -> the dense table of the contraction: entry e goes to column
    rank_e * cells + kernel_index[e] of an int32 [num_out, R * cells] table, rank_e counting the earlier entries of its
    (row, cell), R the largest such count (the filters are repeated R times).  entry_weight: None, or rows -> float
    [E], the entries' weights, scattered into a parallel float table (zero where the table holds the shadow id num_in).
    One host read (none without entries), which also returns the smallest and largest kernel index and the end of the
    row splits: a kernel index outside [0, cells), or splits that do not end at E, raise before anything is scattered
    or weighed.  -> (table, weight table or None, R, rows of the entries, row lengths)."""
    rs = _dev(neighbors_row_splits).to(dev, torch.int64).reshape(-1)
    if rs.numel() < 1:
        raise RuntimeError("%s: neighbors_row_splits must have num_out + 1 elements" % name)
    m = rs.numel() - 1
    lens = rs[1:] - rs[:-1]
    idx = _dev(neighbors_index).to(dev).reshape(-1)
    kidx = _dev(neighbors_kernel_index).to(dev).reshape(-1).long()
    e = idx.numel()
    if kidx.numel() != e:
        raise RuntimeError("%s: neighbors_kernel_index must have one entry per neighbour" % name)
    pos = torch.arange(e, device=dev)
    rows = torch.searchsorted(rs[1:], pos, right=True)
    group = rows * kc + kidx
    order = torch.argsort(group, stable=True)
    g = group[order]
    first = torch.ones(e, dtype=torch.bool, device=dev)
    first[1:] = g[1:] != g[:-1]
    start = torch.cummax(torch.where(first, pos, 0), 0).values
    rank = torch.empty_like(pos)
    rank[order] = pos - start
    reps = 1
    if e:
        top, kmin, kmax, last = (int(v) for v in torch.stack([rank.max(), kidx.min(), kidx.max(), rs[-1]]).cpu())
        if kmin < 0 or kmax >= kc:
            raise RuntimeError("%s: neighbors_kernel_index holds %d, outside [0, %d)" % (name, kmin if kmin < 0 else kmax,
                                                                                      kc))
        if last != e:
            raise RuntimeError("%s: neighbors_row_splits ends at %d, not at the %d neighbour entries" % (name, last, e))
        reps = top + 1
    col = rank * kc + kidx
    table = torch.full((m, reps * kc), num_in, dtype=torch.int32, device=dev)
    table[rows, col] = idx.to(torch.int32)
    wt = None
    if entry_weight is not None:
        wt = torch.zeros((m, reps * kc), dtype=torch.float32, device=dev)
        wt[rows, col] = entry_weight(rows)
    return table, wt, reps, rows, lens


def sparse_conv(filters, inp_features, inp_importance, neighbors_index, neighbors_kernel_index, neighbors_importance,
                neighbors_row_splits, normalize=False, max_temp_mem_MB=64):
    """open3d.ml.torch.ops.sparse_conv (raw op):
        out[o] = (1 / n_o) sum_e nimp_e * iimp_i * filters[kernel_index[e]]^T f[i],   i = neighbors_index[e],
    over the ragged rows of `neighbors_row_splits`; filters [.., Cin, Cout] with the leading dims flattened into the
    kernel index.  Empty importance tensors mean all ones.  Under normalize n_o = sum_e nimp_e * iimp_i (the row length
    without importances; a zero divisor gives 1), otherwise 1.  A row may name one kernel cell several times (a
    radius search over points that are not voxel-unique): see _sparse_table.  One table-mode tensor-core launch, the
    weighted one when an importance is given; one host read (R and the kernel index range)."""
    name = "sparse_conv"
    feat = layers.aligned_rows(_dev(inp_features).to(torch.float32).contiguous())
    w = _sparse_filters(name, filters, feat)
    kc, cout = w.shape[0], w.shape[2]
    dev, num_in = feat.device, feat.shape[0]
    e = neighbors_index.numel()
    iimp = _sparse_importance(name, "inp_importance", inp_importance, num_in, dev)
    nimp = _sparse_importance(name, "neighbors_importance", neighbors_importance, e, dev)
    weighted = iimp is not None or nimp is not None

    def entry_weight(_rows):
        wt = torch.ones(e, dtype=torch.float32, device=dev) if nimp is None else nimp
        if iimp is not None:     # an index outside [0, num_in) is a shadow entry: any weight does
            idx = _dev(neighbors_index).to(dev).reshape(-1).long()
            wt = wt * torch.cat([iimp, iimp.new_zeros(1)])[torch.where((idx >= 0) & (idx < num_in), idx, num_in)]
        return wt
    table, wt, reps, _, lens = _sparse_table(name, neighbors_index, neighbors_kernel_index, neighbors_row_splits,
                                             kc, num_in, dev, entry_weight if weighted else None)
    m = lens.numel()
    out = torch.zeros((m, cout), dtype=torch.float32, device=dev)
    layers.contract_cells(feat, table, layers.pack_cells(w.repeat(reps, 1, 1)), out, entry_weight=wt)
    if normalize and not weighted:
        out = out / lens.clamp_min(1).to(torch.float32).unsqueeze(1)
    elif normalize:
        n_o = wt.sum(1)                       # the weight table holds every entry's weight once, zeros elsewhere
        out = out / torch.where(n_o != 0, n_o, torch.ones_like(n_o)).unsqueeze(1)
    return _back(out, inp_features.device)


def sparse_conv_transpose(filters, out_importance, inp_features, inp_neighbors_index, inp_neighbors_importance_sum,
                          inp_neighbors_row_splits, neighbors_index, neighbors_kernel_index, neighbors_importance,
                          neighbors_row_splits, normalize=False, max_temp_mem_MB=64):
    """open3d.ml.torch.ops.sparse_conv_transpose (raw op), the adjoint of sparse_conv: for output j and the entries e
    of its ragged row (input i = neighbors_index[e]),
        out[j] = oimp_j * sum_e nimp_e * s_i * filters[kernel_index[e]]^T f[i],
    filters [.., Cin, Cout] with the leading dims flattened into the kernel index, inp_features [num_inp, Cin] ->
    [num_out, Cout].  The neighbors_* lists are those of sparse_conv inverted (invert_neighbors_list, with the kernel
    index and importance carried as attributes).  Empty importance tensors mean all ones.  Under normalize
    s_i = 1 / inp_neighbors_importance_sum[i], or 1 / the length of row i of inp_neighbors_row_splits when that sum is
    empty (one of the two is required), 1 for a zero divisor; s_i = 1 without normalize.  inp_neighbors_index is taken
    for signature parity and not read.  One table-mode launch, the weighted one unless every weight is one; one host
    read, as sparse_conv."""
    name = "sparse_conv_transpose"
    feat = layers.aligned_rows(_dev(inp_features).to(torch.float32).contiguous())
    w = _sparse_filters(name, filters, feat)
    kc, cout = w.shape[0], w.shape[2]
    dev, num_in = feat.device, feat.shape[0]
    e, num_out = neighbors_index.numel(), neighbors_row_splits.numel() - 1
    oimp = _sparse_importance(name, "out_importance", out_importance, num_out, dev)
    nimp = _sparse_importance(name, "neighbors_importance", neighbors_importance, e, dev)
    s = None
    if normalize:
        s = _sparse_importance(name, "inp_neighbors_importance_sum", inp_neighbors_importance_sum, num_in, dev)
        if s is None:
            if inp_neighbors_row_splits is None or inp_neighbors_row_splits.numel() == 0:
                raise RuntimeError("%s: normalize needs inp_neighbors_importance_sum or inp_neighbors_row_splits" % name)
            irs = _dev(inp_neighbors_row_splits).to(dev, torch.int64).reshape(-1)
            if irs.numel() != num_in + 1:
                raise RuntimeError("%s: inp_neighbors_row_splits must have num_inp + 1 elements" % name)
            s = (irs[1:] - irs[:-1]).to(torch.float32)
        s = torch.where(s != 0, 1.0 / s, torch.ones_like(s))

    def entry_weight(rows):
        wt = torch.ones(e, dtype=torch.float32, device=dev) if nimp is None else nimp
        if s is not None:        # an index outside [0, num_inp) is a shadow entry: any weight does
            idx = _dev(neighbors_index).to(dev).reshape(-1).long()
            wt = wt * torch.cat([s, s.new_ones(1)])[torch.where((idx >= 0) & (idx < num_in), idx, num_in)]
        return wt if oimp is None else wt * oimp[rows]
    weighted = oimp is not None or nimp is not None or s is not None
    table, wt, reps, _, _ = _sparse_table(name, neighbors_index, neighbors_kernel_index, neighbors_row_splits, kc,
                                          num_in, dev, entry_weight if weighted else None)
    out = torch.zeros((num_out, cout), dtype=torch.float32, device=dev)
    layers.contract_cells(feat, table, layers.pack_cells(w.repeat(reps, 1, 1)), out, entry_weight=wt)
    return _back(out, inp_features.device)
