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


def _splits(row_splits, n, device):
    if row_splits is None:
        return torch.tensor([0, n], dtype=torch.int64, device=device)
    if row_splits.dtype != torch.int64:
        raise RuntimeError("row_splits must be int64")
    return row_splits.to(device).contiguous()


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
    wsb = L.lib().o3dml_voxelize_workspace_bytes(n, batch)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
    L.check(L.lib().o3dml_voxelize(
        L.ptr(points), n, points.stride(0), L.ptr(rs), batch, vs.ctypes.data, rmin.ctypes.data,
        rmax.ctypes.data, int(min(max_points_per_voxel, INT64_MAX)), int(min(max_voxels, INT64_MAX)),
        L.ptr(coords), L.ptr(pidx), L.ptr(vrs), L.ptr(bsp), L.ptr(bid), L.ptr(counts), L.ptr(ws),
        wsb, L.stream()))
    return coords, pidx, vrs, bsp, bid, counts


def voxelize(points, row_splits, voxel_size, points_range_min, points_range_max,
             max_points_per_voxel=INT64_MAX, max_voxels=INT64_MAX):
    """open3d.ml.torch.ops.voxelize -- one device->host read (the voxel count)."""
    was_cuda = points.is_cuda
    coords, pidx, vrs, bsp, _, counts = voxelize_raw(points, row_splits, voxel_size,
                                                     points_range_min, points_range_max,
                                                     max_points_per_voxel, max_voxels)
    m, kept = (int(v) for v in counts.tolist())
    out = VoxelizeResult(coords[:m], pidx[:kept], vrs[:m + 1], bsp)
    return out if was_cuda else VoxelizeResult(*(t.cpu() for t in out))


def ragged_to_dense(values, row_splits, out_col_size, default_value, _add=0):
    """open3d.ml.torch.ops.ragged_to_dense for integer / float32 values of shape [L] or [L, ...]."""
    was_cuda = values.is_cuda
    v = _dev(values).contiguous()
    if v.element_size() not in (4, 8):
        raise RuntimeError("ragged_to_dense: 4- or 8-byte element types only")
    rs = _dev(row_splits)
    if rs.dtype != torch.int64:
        raise RuntimeError("row_splits must be int64")
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
    return out if was_cuda else out.cpu()


def knn_workspace_bytes(num_points, num_queries, batch):
    return L.lib().o3dml_knn_workspace_bytes(num_points, num_queries, batch)


def knn_search_raw(points, points_row_splits, queries, queries_row_splits, k, out_index, out_distance2=None,
                   workspace=None):
    """Sync-free form of knn_search: contiguous CUDA points / queries [N,3] with int64 row splits, dense outputs from
    the caller (out_index int32 or int64 [Nq, k], out_distance2 float32 [Nq, k] or None), and a uint8 workspace of
    at least knn_workspace_bytes, allocated here when none is given."""
    batch = points_row_splits.numel() - 1
    if workspace is None:
        wsb = knn_workspace_bytes(points.shape[0], queries.shape[0], batch)
        workspace = torch.empty((wsb,), dtype=torch.uint8, device=points.device)
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


def knn_search(points, queries, k, points_row_splits=None, queries_row_splits=None,
               index_dtype=torch.int32, metric="L2", ignore_query_point=False,
               return_distances=False, allow_short=False):
    """open3d.ml.torch.ops.knn_search.  Rows ascend by (distance, index) in `metric` (L1, L2, Linf); L2 distances are
    squared, as upstream returns them.  Dense [Nq * k] rows with row splits 0, k, 2k, ...; with ignore_query_point
    (points equal to the query are skipped) a row may hold fewer than k neighbours, and the rows are ragged (one
    device->host read of their total)."""
    m = _metric(metric, "knn_search")
    _index_dtype(index_dtype, "knn_search")
    _check_points(points), _check_points(queries, "queries")
    was_cuda = points.is_cuda
    p, q = _dev(points).contiguous(), _dev(queries).contiguous()
    dev = p.device
    ps, qs = _splits(points_row_splits, p.shape[0], dev), _splits(queries_row_splits, q.shape[0], dev)
    batch = ps.numel() - 1
    if qs.numel() - 1 != batch:
        raise RuntimeError("knn_search: row splits disagree on the batch size")
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
        wsb = L.lib().o3dml_knn_search_metric_workspace_bytes(p.shape[0], nq, batch, k, ig)
        ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
        L.check(L.lib().o3dml_knn_search_metric(L.ptr(p), p.shape[0], L.ptr(ps), L.ptr(q), nq, L.ptr(qs), batch, k, m,
                                                ig, L.ptr(idx), L.is64(idx), L.ptr(d2), L.ptr(rs), L.ptr(total),
                                                L.ptr(ws), wsb, L.stream()))
        if ig:
            t = int(total.item())
            idx, d2 = idx[:t], (d2[:t] if d2 is not None else None)
    out = KnnResult(idx.reshape(-1), rs,
                    d2.reshape(-1) if d2 is not None else torch.empty(0, device=dev))
    return out if was_cuda else KnnResult(*(t.cpu() for t in out))


def _radius_search(name, points, queries, radius, radii, points_row_splits, queries_row_splits, index_dtype, metric,
                   ignore_query_point, return_distances, normalize_distances):
    """Two-phase radius search (count, one device->host read of the total, fill) with one radius (radii None) or
    one per query."""
    m = _metric(metric, name)
    _index_dtype(index_dtype, name)
    _check_points(points), _check_points(queries, "queries")
    was_cuda = points.is_cuda
    p, q = _dev(points).contiguous(), _dev(queries).contiguous()
    dev = p.device
    ps, qs = _splits(points_row_splits, p.shape[0], dev), _splits(queries_row_splits, q.shape[0], dev)
    batch = ps.numel() - 1
    if qs.numel() - 1 != batch:
        raise RuntimeError("%s: row splits disagree on the batch size" % name)
    nq = q.shape[0]
    if radii is not None:
        radii = _dev(torch.as_tensor(radii)).reshape(-1).contiguous()
        if radii.dtype != torch.float32 or radii.numel() != nq:
            raise RuntimeError("%s: radii must be float32 with one radius per query (%d)" % (name, nq))
    ig, norm = 1 if ignore_query_point else 0, 1 if normalize_distances else 0
    nrs = torch.empty((nq + 1,), dtype=torch.int64, device=dev)
    total = torch.zeros((1,), dtype=torch.int64, device=dev)
    wsb = L.lib().o3dml_radius_workspace_bytes(p.shape[0], nq, batch)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
    L.check(L.lib().o3dml_radius_search_count(L.ptr(p), p.shape[0], L.ptr(ps), L.ptr(q), nq, L.ptr(qs), batch,
                                              float(radius), L.ptr(radii), m, ig, L.ptr(nrs), L.ptr(total), L.ptr(ws),
                                              wsb, L.stream()))
    t = int(total.item())
    idx = torch.empty((t,), dtype=index_dtype, device=dev)
    d = torch.empty((t,), dtype=torch.float32, device=dev)
    if t:      # with no neighbour at all there is nothing to fill (and the empty outputs have no address)
        L.check(L.lib().o3dml_radius_search_fill(L.ptr(q), p.shape[0], nq, L.ptr(qs), batch, float(radius),
                                                 L.ptr(radii), m, ig, norm, L.ptr(nrs), L.ptr(idx), L.is64(idx),
                                                 L.ptr(d), L.ptr(ws), wsb, L.stream()))
    out = RadiusResult(idx, nrs, d if return_distances else torch.empty(0, device=dev))
    return out if was_cuda else RadiusResult(*(t_.cpu() for t_ in out))


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
    was_cuda = boxes.is_cuda
    b = _dev(boxes).to(torch.float32).contiguous()
    s = _dev(scores).to(torch.float32).contiguous()
    n = b.shape[0]
    keep = torch.empty((n,), dtype=torch.int64, device=b.device)
    cnt = torch.zeros((1,), dtype=torch.int64, device=b.device)
    wsb = L.lib().o3dml_nms_workspace_bytes(n)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=b.device)
    L.check(L.lib().o3dml_nms(L.ptr(b), L.ptr(s), n, float(nms_overlap_thresh), L.ptr(keep), L.ptr(cnt), L.ptr(ws),
                              wsb, L.stream()))
    out = keep[:int(cnt.item())]
    return out if was_cuda else out.cpu()


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
    if row_splits.dtype != torch.int64:
        raise RuntimeError("row_splits must be int64")
    was_cuda = values.is_cuda
    v = _dev(values).to(torch.float32).contiguous()
    rs = _dev(row_splits).contiguous()
    rows = rs.numel() - 1
    out = torch.empty((max(rows, 0),), dtype=torch.float32, device=v.device)
    L.check(L.lib().o3dml_reduce_subarrays_sum(L.ptr(v), L.ptr(rs), rows, L.ptr(out), L.stream()))
    out = out.to(values.dtype)
    return out if was_cuda else out.cpu()


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
    was_cuda = positions.is_cuda
    pts = _dev(positions).contiguous()
    feats = _dev(features).to(torch.float32).contiguous()
    if feats.dim() != 2 or feats.shape[0] != pts.shape[0]:
        raise RuntimeError("voxel_pooling: features must have shape [N, C]")
    if pts.shape[0] == 0:
        out = VoxelPoolingResult(pts.new_zeros((0, 3)), feats.new_zeros((0, feats.shape[1])))
        return out if was_cuda else VoxelPoolingResult(*(t.cpu() for t in out))
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
    out = VoxelPoolingResult(op, of)
    return out if was_cuda else VoxelPoolingResult(*(t.cpu() for t in out))


_CCONV_MAPPING = {"identity": 0, "ball_to_cube_radial": 1}
_CCONV_INTERP = {"nearest_neighbor": 0, "linear": 1, "linear_border": 2}


def continuous_conv(filters, out_positions, extents, offset, inp_positions, inp_features, inp_importance,
                    neighbors_index, neighbors_importance, neighbors_row_splits, align_corners=False,
                    coordinate_mapping="ball_to_cube_radial", normalize=False, interpolation="linear",
                    max_temp_mem_MB=64):
    """open3d.ml.torch.ops.continuous_conv (raw op; contract in csrc/cconv.cu).  filters [Sz, Sy, Sx, Cin, Cout];
    empty importance tensors mean "all ones"; extents [1] or [num_out]."""
    if coordinate_mapping not in _CCONV_MAPPING:
        raise RuntimeError("continuous_conv: coordinate_mapping '%s' is not implemented (identity, ball_to_cube_radial)"
                           % coordinate_mapping)
    if interpolation not in _CCONV_INTERP:
        raise RuntimeError("continuous_conv: unknown interpolation '%s'" % interpolation)
    if filters.dim() != 5:
        raise RuntimeError("continuous_conv: filters must have shape [Sz, Sy, Sx, Cin, Cout]")
    was_cuda = inp_features.is_cuda
    f = _dev(filters).to(torch.float32).contiguous()
    op, ip = _dev(out_positions).to(torch.float32).contiguous(), _dev(inp_positions).to(torch.float32).contiguous()
    feat = _dev(inp_features).to(torch.float32).contiguous()
    ext = _dev(torch.as_tensor(extents, dtype=torch.float32).reshape(-1)).contiguous()
    if ext.numel() not in (1, op.shape[0]):
        raise RuntimeError("continuous_conv: extents must have 1 or num_out elements")
    off = np.ascontiguousarray(torch.as_tensor(offset).detach().cpu().numpy(), dtype=np.float32).reshape(3)
    imp = None if inp_importance is None or inp_importance.numel() == 0 else _dev(inp_importance).float().contiguous()
    nimp = (None if neighbors_importance is None or neighbors_importance.numel() == 0
            else _dev(neighbors_importance).float().contiguous())
    idx = _dev(neighbors_index).contiguous()
    if idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("continuous_conv: neighbors_index must be int32 or int64")
    rs = _dev(neighbors_row_splits).to(torch.int64).contiguous()
    if rs.numel() != op.shape[0] + 1:
        raise RuntimeError("continuous_conv: neighbors_row_splits must have num_out + 1 elements")
    sz, sy, sx, cin, cout = f.shape
    if feat.shape[1] != cin:
        raise RuntimeError("continuous_conv: feature channels do not match the filter")
    out = torch.empty((op.shape[0], cout), dtype=torch.float32, device=f.device)
    L.check(L.lib().o3dml_continuous_conv(
        L.ptr(f), sx, sy, sz, cin, cout, L.ptr(op), op.shape[0], L.ptr(ext), 1 if ext.numel() > 1 else 0,
        off.ctypes.data, L.ptr(ip), L.ptr(feat), ip.shape[0], L.ptr(imp), L.ptr(idx),
        L.is64(idx), L.ptr(nimp), L.ptr(rs), 1 if align_corners else 0,
        _CCONV_MAPPING[coordinate_mapping], 1 if normalize else 0, _CCONV_INTERP[interpolation], L.ptr(out), L.stream()))
    return out if was_cuda else out.cpu()


InvertNeighborsListResult = collections.namedtuple(
    "InvertNeighborsListResult", "neighbors_index neighbors_row_splits neighbors_attributes")


def invert_neighbors_list(num_points, inp_neighbors_index, inp_neighbors_row_splits, inp_neighbors_attributes):
    """open3d.ml.torch.ops.invert_neighbors_list: num_inp rows of ids in [0, num_points) -> num_points rows of the
    input rows that contain each id, once per occurrence, by (input row, position in it): a stable sort by id.  Ids out
    of range are dropped (they follow the last row; neighbors_row_splits[-1] counts the entries kept).  The attributes
    ([E, ...], any dtype) are permuted the same way; an empty attributes tensor stays empty.  No host read."""
    was_cuda = inp_neighbors_index.is_cuda
    idx = _dev(inp_neighbors_index).reshape(-1).contiguous()
    if idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("invert_neighbors_list: inp_neighbors_index must be int32 or int64")
    if inp_neighbors_row_splits.dtype != torch.int64:
        raise RuntimeError("row_splits must be int64")
    rs = _dev(inp_neighbors_row_splits).contiguous()
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
    wsb = L.lib().o3dml_invert_neighbors_list_workspace_bytes(e)
    ws = torch.empty((wsb,), dtype=torch.uint8, device=dev)
    L.check(L.lib().o3dml_invert_neighbors_list(num_points, L.ptr(idx), L.is64(idx), L.ptr(rs), num_inp, e,
                                                L.ptr(out_idx), L.ptr(out_rs), L.ptr(perm), L.ptr(ws), wsb,
                                                L.stream()))
    out_attrs = _dev(attrs)[perm] if attrs.numel() else attrs
    if was_cuda:
        return InvertNeighborsListResult(out_idx, out_rs, out_attrs)
    return InvertNeighborsListResult(out_idx.cpu(), out_rs.cpu(), out_attrs.cpu())


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
    if coordinate_mapping not in _CCONV_MAPPING:
        raise RuntimeError("%s: coordinate_mapping '%s' is not implemented (identity, ball_to_cube_radial)"
                           % (name, coordinate_mapping))
    if interpolation not in _CCONV_INTERP:
        raise RuntimeError("%s: unknown interpolation '%s'" % (name, interpolation))
    if filters.dim() != 5:
        raise RuntimeError("%s: filters must have shape [Sz, Sy, Sx, Cin, Cout]" % name)
    was_cuda = inp_features.is_cuda
    f = _dev(filters).to(torch.float32).contiguous()
    op, ip = _dev(out_positions).to(torch.float32).contiguous(), _dev(inp_positions).to(torch.float32).contiguous()
    feat = _dev(inp_features).to(torch.float32).contiguous()
    num_out, num_inp = op.shape[0], ip.shape[0]
    ext = _dev(torch.as_tensor(extents, dtype=torch.float32).reshape(-1)).contiguous()
    if ext.numel() != 1 and (ext.numel() != num_inp or num_inp == 0):
        raise RuntimeError("%s: extents must have 1 or num_inp elements" % name)
    off = np.ascontiguousarray(torch.as_tensor(offset).detach().cpu().numpy(), dtype=np.float32).reshape(3)

    def opt(t, n, what):
        if t is None or t.numel() == 0:
            return None
        t = _dev(t).float().reshape(-1).contiguous()
        if t.numel() != n:
            raise RuntimeError("%s: %s must be empty or have %d elements" % (name, what, n))
        return t
    oimp = opt(out_importance, num_out, "out_importance")
    isum = opt(inp_neighbors_importance_sum, num_inp, "inp_neighbors_importance_sum")
    nimp = opt(neighbors_importance, neighbors_index.numel(), "neighbors_importance")
    irs = None
    if inp_neighbors_row_splits is not None and inp_neighbors_row_splits.numel():
        irs = _dev(inp_neighbors_row_splits).to(torch.int64).contiguous()
        if irs.numel() != num_inp + 1:
            raise RuntimeError("%s: inp_neighbors_row_splits must have num_inp + 1 elements" % name)
    idx = _dev(neighbors_index).contiguous()
    if idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("%s: neighbors_index must be int32 or int64" % name)
    rs = _dev(neighbors_row_splits).to(torch.int64).contiguous()
    if rs.numel() != num_out + 1:
        raise RuntimeError("%s: neighbors_row_splits must have num_out + 1 elements" % name)
    sz, sy, sx, cin, cout = f.shape
    if feat.dim() != 2 or feat.shape[0] != num_inp or feat.shape[1] != cin:
        raise RuntimeError("%s: feature channels do not match the filter" % name)
    out = torch.empty((num_out, cout), dtype=torch.float32, device=f.device)
    L.check(L.lib().o3dml_continuous_conv_transpose(
        L.ptr(f), sx, sy, sz, cin, cout, L.ptr(op), num_out, L.ptr(oimp), L.ptr(ext), 1 if ext.numel() > 1 else 0,
        off.ctypes.data, L.ptr(ip), L.ptr(feat), num_inp, L.ptr(isum), L.ptr(irs), L.ptr(idx), L.is64(idx),
        L.ptr(nimp), L.ptr(rs), 1 if align_corners else 0, _CCONV_MAPPING[coordinate_mapping], 1 if normalize else 0,
        _CCONV_INTERP[interpolation], L.ptr(out), L.stream()))
    return out if was_cuda else out.cpu()


def sparse_conv(filters, inp_features, inp_importance, neighbors_index, neighbors_kernel_index, neighbors_importance,
                neighbors_row_splits, normalize=False, max_temp_mem_MB=64):
    """open3d.ml.torch.ops.sparse_conv (raw op): out[o] = sum_j filters[kernel_index[j]]^T f[neighbors_index[j]] over
    the ragged rows of `neighbors_row_splits`; filters [.., Cin, Cout] with the leading dims flattened into the kernel
    index.  Runs as gathered tensor-core GEMMs over a dense [num_out, kernel_cells] table (one neighbour per cell)."""
    if (inp_importance is not None and inp_importance.numel()) or \
            (neighbors_importance is not None and neighbors_importance.numel()):
        raise RuntimeError("sparse_conv: importance is not implemented")
    was_cuda = inp_features.is_cuda
    w = filters.detach().float().cpu()
    cin, cout = w.shape[-2], w.shape[-1]
    w = w.reshape(-1, cin, cout)
    kc = w.shape[0]
    feat = _dev(inp_features).to(torch.float32).contiguous()
    rs = _dev(neighbors_row_splits).to(torch.int64)
    m = rs.numel() - 1
    lens = rs[1:] - rs[:-1]
    rows = torch.repeat_interleave(torch.arange(m, device=feat.device), lens)
    table = torch.full((m, kc), feat.shape[0], dtype=torch.int32, device=feat.device)
    table[rows, _dev(neighbors_kernel_index).long()] = _dev(neighbors_index).to(torch.int32)
    out = torch.zeros((m, cout), dtype=torch.float32, device=feat.device)
    layers.contract_cells(feat, table, layers.pack_cell_groups(w), out)
    if normalize:
        out = out / lens.clamp_min(1).to(torch.float32).unsqueeze(1)
    return out if was_cuda else out.cpu()
