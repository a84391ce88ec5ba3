"""Seeded calls of the C-ABI entries (include/o3dml_b200.h) and the case tables of the ABI contract tests: LAUNCH_CASES,
EXPECTED_LAUNCHES and EXPECTED_KERNEL (tests/test_gpu_launch_count.py), WORKSPACE_CASES (tests/test_gpu_workspace.py)
and REFUSAL_ROWS (tests/test_workspace.py).  tests/test_abi.py checks that these tables cover every entry the library
exports, so a new entry is added here.  Each builder allocates everything its call needs on the GPU; an entry that takes a workspace
is built as a WsCase whose `run` takes the workspace as an argument, so that a test can choose where the workspace lies
and how large it is said to be.  Importing this module needs no GPU."""
import json
import os
import tempfile

import numpy as np
import torch

from open3d_ml_b200 import _lib as L, layers as LY
from oracle import ops as O, search as S
import cconv_transpose_oracle as R


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


def boxes(n, seed):
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * 20
    wh = torch.rand(n, 2, generator=g) * 3 + 0.5
    return torch.cat([xy, xy + wh, torch.rand(n, 1, generator=g)], 1).cuda()


def counted_and_traced(call):
    """(counter delta, names of the kernel activities in the trace) of one call."""
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        n0 = L.lib().o3dml_launch_count()
        rc = call()
        n1 = L.lib().o3dml_launch_count()
        torch.cuda.synchronize()
    if isinstance(rc, int):
        L.check(rc)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return n1 - n0, [e["name"] for e in events if e.get("ph") == "X" and e.get("cat") == "kernel"]


class WsCase:
    """sizing, wsb: the entry's *_workspace_bytes function and what it returns for the case; run(ws, nbytes): the call
    with its workspace at device address ws, returning the entry's status; outputs: the tensors the call writes;
    reference: None, or a function giving the oracle's value of each output in order (of the fill outputs after
    them, for a two-phase case)."""

    def __init__(self, sizing, sizing_args, run, outputs, reference=None):
        self.sizing, self.wsb = sizing, getattr(L.lib(), sizing)(*sizing_args)
        self.run, self.outputs, self.reference = run, outputs, reference

    def with_own_workspace(self):
        """The call as a closure over a workspace of its own, wsb bytes."""
        ws = torch.empty(self.wsb, dtype=torch.uint8).cuda()
        return lambda: self.run(L.ptr(ws), self.wsb)


def after_count(case):
    """The fill of a two-phase case, as a closure, after its count has run over a workspace of its own."""
    ws = torch.empty(case.wsb, dtype=torch.uint8).cuda()
    L.check(case.run(L.ptr(ws), case.wsb))
    case.prepare_fill()
    return lambda: case.fill(L.ptr(ws), case.wsb)


# ------------------------------------------------------------------------------------- entries with a workspace
def voxelize_case(splits=(0, 250, 500), voxel=0.5, max_voxels=1000, seed=1):
    n, batch = splits[-1], len(splits) - 1
    pts = (torch.rand(n, 4, generator=torch.Generator().manual_seed(seed)) * 4).cuda()
    rs = torch.tensor(splits, dtype=torch.int64).cuda()
    host = [np.full(3, v, np.float32) for v in (voxel, 0.0, 4.0)]      # voxel size, range min, range max
    out = dict(coords=torch.empty(n, 3, dtype=torch.int32).cuda(), pidx=torch.empty(n, dtype=torch.int64).cuda(),
               vrs=torch.empty(n + 1, dtype=torch.int64).cuda(), bsp=torch.empty(batch + 1, dtype=torch.int64).cuda(),
               bid=torch.empty(n, dtype=torch.int32).cuda(), counts=torch.empty(2, dtype=torch.int64).cuda())

    def run(ws, nbytes):
        return L.lib().o3dml_voxelize(L.ptr(pts), n, pts.stride(0), L.ptr(rs), batch, host[0].ctypes.data,
                                      host[1].ctypes.data, host[2].ctypes.data, 32, max_voxels, L.ptr(out["coords"]),
                                      L.ptr(out["pidx"]), L.ptr(out["vrs"]), L.ptr(out["bsp"]), L.ptr(out["bid"]),
                                      L.ptr(out["counts"]), ws, nbytes, L.stream())
    case = WsCase("o3dml_voxelize_workspace_bytes", (n, batch), run, list(out.values()))
    case.pts, case.out = pts, out
    return case


def knn_case(p_splits=(0, 500), q_splits=(0, 300), k=8):
    num_points, num_queries, batch = p_splits[-1], q_splits[-1], len(p_splits) - 1
    p, q = rnd(num_points, 3, seed=1), rnd(num_queries, 3, seed=2)
    ps = torch.tensor(p_splits, dtype=torch.int64).cuda()
    qs = torch.tensor(q_splits, dtype=torch.int64).cuda()
    idx, d2 = torch.empty(num_queries, k, dtype=torch.int32).cuda(), torch.empty(num_queries, k).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_knn_search(L.ptr(p), num_points, L.ptr(ps), L.ptr(q), num_queries, L.ptr(qs), batch, k,
                                        L.ptr(idx), 0, L.ptr(d2), ws, nbytes, L.stream())
    return WsCase("o3dml_knn_workspace_bytes", (num_points, num_queries, batch), run, [idx, d2])


def radius_case(p_splits=(0, 200, 400), q_splits=(0, 100, 200), radius=0.8):
    """run is o3dml_radius_count.  After a count, prepare_fill() allocates the rows it sized; fill(ws, nbytes) then
    runs o3dml_radius_fill into them (fill_outputs) over the same workspace."""
    num_points, num_queries, batch = p_splits[-1], q_splits[-1], len(p_splits) - 1
    p, q = rnd(num_points, 3, seed=3), rnd(num_queries, 3, seed=4)
    ps = torch.tensor(p_splits, dtype=torch.int64).cuda()
    qs = torch.tensor(q_splits, dtype=torch.int64).cuda()
    nrs, total = torch.empty(num_queries + 1, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def count(ws, nbytes):
        return L.lib().o3dml_radius_count(L.ptr(p), num_points, L.ptr(ps), L.ptr(q), num_queries, L.ptr(qs), batch,
                                          radius, L.ptr(nrs), L.ptr(total), ws, nbytes, L.stream())
    case = WsCase("o3dml_radius_workspace_bytes", (num_points, num_queries, batch), count, [nrs, total])

    def prepare_fill():
        t = int(total.item())
        case.fill_outputs = [torch.zeros(t, dtype=torch.int32).cuda(), torch.zeros(t).cuda()]

    def fill(ws, nbytes):
        idx, d2 = case.fill_outputs
        return L.lib().o3dml_radius_fill(L.ptr(q), num_points, num_queries, L.ptr(qs), batch, radius, L.ptr(nrs),
                                         L.ptr(idx), L.ptr(d2), ws, nbytes, L.stream())
    case.prepare_fill, case.fill = prepare_fill, fill
    return case


def search_inputs(num_points=2000, num_queries=900, batch_splits=((0, 1200, 2000), (0, 500, 900))):
    """Host points, queries, their splits and one radius per query of the general searches' cases."""
    rng = np.random.default_rng(9)
    p = rng.random((num_points, 3)).astype(np.float32)
    q = rng.random((num_queries, 3)).astype(np.float32)
    radii = rng.uniform(0.02, 0.08, num_queries).astype(np.float32)
    return p, q, np.array(batch_splits[0], np.int64), np.array(batch_splits[1], np.int64), radii


def radius_search_case():
    """o3dml_radius_search_count + _fill with one radius per query, L-infinity, ignore_query_point,
    normalize_distances and int64 ids, shaped as radius_case."""
    p, q, ps, qs, radii = search_inputs()
    num_points, num_queries, batch = len(p), len(q), len(ps) - 1
    dp, dq, dps, dqs, dradii = (torch.from_numpy(a).cuda() for a in (p, q, ps, qs, radii))
    nrs, total = torch.empty(num_queries + 1, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def count(ws, nbytes):
        return L.lib().o3dml_radius_search_count(L.ptr(dp), num_points, L.ptr(dps), L.ptr(dq), num_queries, L.ptr(dqs),
                                                 batch, 0.0, L.ptr(dradii), 2, 1, L.ptr(nrs), L.ptr(total), ws, nbytes,
                                                 L.stream())

    def reference():
        idx, rs, d = S.c_search_radius(p, q, 0.0, radii, ps, qs, 2, True, True)
        return [rs, rs[-1:], idx, d]
    case = WsCase("o3dml_radius_workspace_bytes", (num_points, num_queries, batch), count, [nrs, total], reference)

    def prepare_fill():
        t = int(total.item())
        case.fill_outputs = [torch.zeros(t, dtype=torch.int64).cuda(), torch.zeros(t).cuda()]

    def fill(ws, nbytes):
        idx, d = case.fill_outputs
        return L.lib().o3dml_radius_search_fill(L.ptr(dq), num_points, num_queries, L.ptr(dqs), batch, 0.0,
                                                L.ptr(dradii), 2, 1, 1, L.ptr(nrs), L.ptr(idx), 1, L.ptr(d), ws,
                                                nbytes, L.stream())
    case.prepare_fill, case.fill = prepare_fill, fill
    return case


def knn_metric_case(k=12):
    """o3dml_knn_search_metric in L1 with ignore_query_point and int64 ids: the rows go back to back, so idx and d
    hold `total` entries at their front."""
    p, q, ps, qs, _ = search_inputs()
    num_points, num_queries, batch = len(p), len(q), len(ps) - 1
    dp, dq, dps, dqs = (torch.from_numpy(a).cuda() for a in (p, q, ps, qs))
    idx, d = torch.empty(num_queries * k, dtype=torch.int64).cuda(), torch.empty(num_queries * k).cuda()
    rs, total = torch.empty(num_queries + 1, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_knn_search_metric(L.ptr(dp), num_points, L.ptr(dps), L.ptr(dq), num_queries, L.ptr(dqs),
                                               batch, k, 1, 1, L.ptr(idx), 1, L.ptr(d), L.ptr(rs), L.ptr(total), ws,
                                               nbytes, L.stream())

    def reference():
        ref_idx, ref_d, n = S.c_search_knn(p, q, k, ps, qs, 1, True)
        keep = np.arange(k)[None, :] < n[:, None]
        ref_rs = np.concatenate([[0], np.cumsum(n)])
        return [ref_idx[keep], ref_d[keep], ref_rs, ref_rs[-1:]]
    return WsCase("o3dml_knn_search_metric_workspace_bytes", (num_points, num_queries, batch, k, 1), run,
                  [idx, d, rs, total], reference)


def sparse_conv_case(num_in, num_out=100):
    ip = torch.randint(0, 8, (num_in, 3), generator=torch.Generator().manual_seed(6)).float().cuda()
    op = torch.randint(0, 8, (num_out, 3), generator=torch.Generator().manual_seed(7)).float().cuda()
    off, ks = np.zeros(3, np.float32), np.full(3, 3, np.int32)
    nbr, cnt = torch.empty(num_out, 27, dtype=torch.int32).cuda(), torch.empty(num_out, dtype=torch.int32).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_sparse_conv_neighbors(L.ptr(ip), num_in, L.ptr(op), num_out, 1.0, off.ctypes.data,
                                                   ks.ctypes.data, 0, L.ptr(nbr), L.ptr(cnt), ws, nbytes, L.stream())
    return WsCase("o3dml_sparse_conv_workspace_bytes", (num_in,), run, [nbr, cnt])


def invert_case(num_entries, num_points=3000, rows=None, seed=48):
    """o3dml_invert_neighbors_list over num_entries ids in rows of up to 8, a tenth of them out of range."""
    rng = np.random.default_rng(seed)
    rows = rows if rows is not None else max(1, num_entries // 4)
    lens = np.zeros(rows, np.int64)
    if num_entries:
        cuts = np.sort(rng.integers(0, num_entries + 1, rows - 1))
        lens = np.diff(np.concatenate([[0], cuts, [num_entries]]))
    splits = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(-1, num_points + num_points // 10, num_entries).astype(np.int32)
    d_idx, d_splits = torch.from_numpy(idx).cuda(), torch.from_numpy(splits).cuda()
    out = dict(idx=torch.empty(num_entries, dtype=torch.int32).cuda(),
               rs=torch.empty(num_points + 1, dtype=torch.int64).cuda(),
               perm=torch.empty(num_entries, dtype=torch.int64).cuda())

    def run(ws, nbytes):
        return L.lib().o3dml_invert_neighbors_list(num_points, L.ptr(d_idx), 0, L.ptr(d_splits), rows, num_entries,
                                                   L.ptr(out["idx"]), L.ptr(out["rs"]), L.ptr(out["perm"]), ws,
                                                   nbytes, L.stream())
    return WsCase("o3dml_invert_neighbors_list_workspace_bytes", (num_entries,), run, list(out.values()),
                  lambda: list(R.invert_neighbors_list(num_points, idx.astype(np.int64), splits)))


def nms_case(n=300):
    b, s = boxes(n, 12), rnd(n, seed=13)
    keep, cnt = torch.empty(n, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_nms(L.ptr(b), L.ptr(s), n, 0.5, L.ptr(keep), L.ptr(cnt), ws, nbytes, L.stream())
    return WsCase("o3dml_nms_workspace_bytes", (n,), run, [keep, cnt])


def pp_detect_case(select):
    B, H, W, A, C = 2, 6, 5, 2, 3
    nms_pre = 20 if select else 100          # select: H * W * A = 60 rows > nms_pre
    cls, reg, dr = rnd(B, A * C, H, W, seed=16), rnd(B, A * 7, H, W, seed=17) * 0.1, rnd(B, A * 2, H, W, seed=18)
    g = torch.Generator().manual_seed(19)
    anchors = torch.cat([torch.rand(H * W * A, 3, generator=g) * 20, torch.rand(H * W * A, 3, generator=g) + 1,
                         torch.rand(H * W * A, 1, generator=g)], 1).cuda()
    K = min(nms_pre, H * W * A)
    bx, sc = torch.empty(B, C * K, 7).cuda(), torch.empty(B, C * K).cuda()
    lab, cnt = torch.empty(B, C * K, dtype=torch.int64).cuda(), torch.empty(B, dtype=torch.int64).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_pp_detect(L.ptr(cls), cls.stride(0), L.ptr(reg), reg.stride(0), L.ptr(dr), dr.stride(0),
                                       B, H, W, A, C, L.ptr(anchors), nms_pre, 0.1, 0.78, L.ptr(bx), L.ptr(sc),
                                       L.ptr(lab), L.ptr(cnt), ws, nbytes, L.stream())
    return WsCase("o3dml_pp_detect_workspace_bytes", (B, H, W, A, C, nms_pre), run, [bx, sc, lab, cnt])


# ------------------------------------------------------------------------------------- entries without a workspace
# Each case_* builder returns the call: a closure that only enters the library, either directly (returning the entry's
# status) or through the _lib wrapper that picks the dense kernel and checks.

def voxelize_inputs():
    case = voxelize_case()
    return case.pts, case.out, case.with_own_workspace()


def case_ragged_to_dense(dtype):
    v = torch.arange(100, dtype=dtype).cuda()
    rs = torch.tensor([0, 30, 30, 100], dtype=torch.int64).cuda()
    out = torch.empty(3, 40, dtype=dtype).cuda()
    return lambda: L.lib().o3dml_ragged_to_dense(L.ptr(v), v.element_size(), 1, L.ptr(rs), 3, 40, -1, 0, L.ptr(out),
                                                 L.stream())


def case_voxel_reduce(labels):
    pts, vox, call = voxelize_inputs()
    L.check(call())
    n = pts.shape[0]
    lab = torch.randint(0, 5, (n,), dtype=torch.int32).cuda() if labels else None
    op, of = torch.empty(n, 3).cuda(), torch.empty(n, 4).cuda()
    ol = torch.empty(n, dtype=torch.int32).cuda()
    return lambda: L.lib().o3dml_voxel_reduce(L.ptr(pts), pts.stride(0), L.ptr(pts), 4, pts.stride(0), L.ptr(lab),
                                              L.ptr(vox["vrs"]), L.ptr(vox["pidx"]), L.ptr(vox["counts"]), n, 0, 1,
                                              L.ptr(op), L.ptr(of), L.ptr(ol) if labels else None, L.stream())


def case_reduce_subarrays_sum():
    v = rnd(100, seed=5)
    rs = torch.tensor([0, 10, 10, 55, 100], dtype=torch.int64).cuda()
    out = torch.empty(4).cuda()
    return lambda: L.lib().o3dml_reduce_subarrays_sum(L.ptr(v), L.ptr(rs), 4, L.ptr(out), L.stream())


def case_continuous_conv():
    m, n, cin, cout = 50, 80, 4, 8
    f = rnd(2, 2, 2, cin, cout, seed=8)
    op, ip, feat = rnd(m, 3, seed=9), rnd(n, 3, seed=10), rnd(n, cin, seed=11)
    ext = torch.tensor([1.0]).cuda()
    off = np.zeros(3, np.float32)
    idx = torch.randint(0, n, (m * 5,), dtype=torch.int32).cuda()
    rs = torch.arange(0, m * 5 + 1, 5, dtype=torch.int64).cuda()
    out = torch.empty(m, cout).cuda()
    return lambda: L.lib().o3dml_continuous_conv(L.ptr(f), 2, 2, 2, cin, cout, L.ptr(op), m, L.ptr(ext), 0,
                                                 off.ctypes.data, L.ptr(ip), L.ptr(feat), n, None, L.ptr(idx), 0, None,
                                                 L.ptr(rs), 0, 0, 0, 1, L.ptr(out), L.stream())


def case_continuous_conv_transpose():
    """The inverted lists of the outputs within 0.25 of each input, normalized by the forward list lengths."""
    rng = np.random.default_rng(49)
    n, m, cin, cout = 80, 50, 4, 8
    ipn, opn = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    fidx, fsplits, _ = O.c_radius(opn, ipn, 0.25)
    tidx, tsplits, _ = R.invert_neighbors_list(m, fidx, fsplits)
    f = torch.from_numpy(rng.standard_normal((2, 2, 2, cin, cout)).astype(np.float32)).cuda()
    feat = torch.from_numpy(rng.standard_normal((n, cin)).astype(np.float32)).cuda()
    o, i, ext = torch.from_numpy(opn).cuda(), torch.from_numpy(ipn).cuda(), torch.tensor([0.5]).cuda()
    off = np.zeros(3, np.float32)
    idx, rs = torch.from_numpy(tidx.astype(np.int32)).cuda(), torch.from_numpy(tsplits).cuda()
    fs = torch.from_numpy(fsplits).cuda()
    out = torch.empty(m, cout).cuda()
    return lambda: L.lib().o3dml_continuous_conv_transpose(
        L.ptr(f), 2, 2, 2, cin, cout, L.ptr(o), m, None, L.ptr(ext), 0, off.ctypes.data, L.ptr(i), L.ptr(feat), n,
        None, L.ptr(fs), L.ptr(idx), 0, None, L.ptr(rs), 1, 1, 1, 1, L.ptr(out), L.stream())


def case_iou_matrix():
    a, b = boxes(40, 14), boxes(30, 15)
    out = torch.empty(40, 30).cuda()
    return lambda: L.lib().o3dml_iou_matrix(L.ptr(a), 40, L.ptr(b), 30, 0, L.ptr(out), L.stream())


def case_pfn_scatter():
    pts, vox, call = voxelize_inputs()
    L.check(call())
    n = pts.shape[0]
    wt, s, t = rnd(16, 64, seed=20), torch.ones(64).cuda(), torch.zeros(64).cuda()
    feat, canvas = torch.empty(n, 64).cuda(), torch.zeros(2, 8, 8, 64).cuda()
    return lambda: L.lib().o3dml_pp_pfn_scatter(L.ptr(pts), pts.stride(0), 4, L.ptr(vox["coords"]), L.ptr(vox["vrs"]),
                                                L.ptr(vox["pidx"]), L.ptr(vox["bid"]), L.ptr(vox["counts"]), n,
                                                L.ptr(wt), L.ptr(s), L.ptr(t), 64, 0.5, 0.5, 0.0, 0.0, 8, 8, 32,
                                                L.ptr(feat), L.ptr(canvas), 0, L.stream())


def case_pfn2_scatter():
    pts, vox, call = voxelize_inputs()
    L.check(call())
    n = pts.shape[0]
    w0, s0, t0 = rnd(9, 32, seed=35), torch.ones(32).cuda(), torch.zeros(32).cuda()
    w1, s1, t1 = rnd(64, 64, seed=36), torch.ones(64).cuda(), torch.zeros(64).cuda()
    feat, canvas = torch.empty(n, 64).cuda(), torch.zeros(2, 8, 8, 64).cuda()
    return lambda: L.lib().o3dml_pp_pfn2_scatter(L.ptr(pts), pts.stride(0), 4, L.ptr(vox["coords"]),
                                                 L.ptr(vox["vrs"]), L.ptr(vox["pidx"]), L.ptr(vox["bid"]),
                                                 L.ptr(vox["counts"]), n, L.ptr(w0), L.ptr(s0), L.ptr(t0), L.ptr(w1),
                                                 L.ptr(s1), L.ptr(t1), 64, 0.5, 0.5, 0.0, 0.0, 8, 8, 32, L.ptr(feat),
                                                 L.ptr(canvas), 0, L.stream())


def case_linear(kind):
    """kind: "simt" (fp32 [K, Cout] weight), "tc" (K = 64 packed weight), "rows_small" (8 -> 8 packed weight)."""
    k = 64 if kind == "tc" else 8
    x, w = rnd(1000, k, seed=21), rnd(k, 8, seed=22)
    weight = w if kind == "simt" else L.pack_linear(w)
    out = torch.empty(1000, 8).cuda()
    src = [L.make_src(x)]
    return lambda: L.linear(src, weight, out, act="relu")


def case_conv3x3(tc):
    x, w = rnd(2, 9, 7, 32, seed=23), rnd(9 * 32, 16, seed=24)
    weight = L.pack_linear(w) if tc else w
    out = torch.empty(2, 5, 4, 16).cuda()
    return lambda: L.conv3x3(x, weight, out, stride=2, act="relu")


def case_deconv(tc):
    x, w = rnd(2, 4, 5, 8, seed=25), rnd(8, 4 * 16, seed=26)
    weight = L.pack_linear(w) if tc else w
    out = torch.empty(2, 8, 10, 16).cuda()
    return lambda: L.deconv(x, weight, out, stride=2, act="relu")


def lfa_inputs(d, B=2, N=300, seed=27):
    g = torch.Generator().manual_seed(seed)
    h = d // 2
    coords = (torch.rand(B * N, 3, generator=g) * 10).cuda()
    nidx = torch.randint(0, N, (B, N, 16), generator=g).cuda()
    feat = torch.randn(B * N, h, generator=g).cuda()
    w10, s10, t10 = (torch.randn(10, h, generator=g) * 0.3).cuda(), torch.ones(h).cuda(), torch.zeros(h).cuda()
    wl2 = torch.randn(h, h, generator=g) / h ** 0.5
    ws = torch.randn(d, d, generator=g) / d ** 0.5
    agg = torch.empty(B * N, d).cuda()
    return coords, nidx, feat, w10, s10, t10, wl2, ws, torch.zeros(d).cuda(), agg


def case_lfa(kind):
    d = 16 if kind == "lfa16" else 32
    coords, nidx, feat, w10, s10, t10, wl2, ws, bs, agg = lfa_inputs(d)
    wl2t, wst = wl2.t().contiguous().cuda(), ws.t().contiguous().cuda()
    B, N = 2, 300
    if kind == "simt":
        return lambda: L.lib().o3dml_randla_lfa_pool(2, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                                     L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(wl2t), L.ptr(s10),
                                                     L.ptr(t10), L.ptr(wst), L.ptr(bs), L.ptr(agg), L.stream())
    if kind == "tc":
        img_l2, img_s = L.pack_operand_image(wl2), L.pack_operand_image(ws)
        return lambda: L.lib().o3dml_randla_lfa_pool_tc(2, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                                        L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(img_l2), L.ptr(wl2t),
                                                        L.ptr(s10), L.ptr(t10), L.ptr(img_s), L.ptr(agg), L.stream())
    hw = L.pack_lfa16_weights(w10, s10, t10, wl2t, s10, t10, wst, bs)
    return lambda: L.lib().o3dml_randla_lfa16_pool(2, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                                   hw.data_ptr(), L.ptr(agg), L.stream())


def case_randla_tail():
    rows, classes = 500, 13
    skip, coarse = rnd(rows, 32, seed=28), rnd(125, 32, seed=29)
    idx = torch.randint(0, 125, (rows,), generator=torch.Generator().manual_seed(30)).cuda()
    g = torch.Generator().manual_seed(31)
    ws = [torch.randn(k, n, generator=g) / k ** 0.5 for k, n in [(64, 32), (32, 64), (64, 32), (32, classes)]]
    img = L.pack_tail_image(ws, [32, 64, 32, 32]).cuda()
    scale, shift = torch.ones(4, 64), torch.zeros(4, 64)
    out = torch.empty(rows, classes).cuda()
    return lambda: L.lib().o3dml_randla_tail(L.ptr(skip), 32, L.ptr(coarse), 32, 125, L.ptr(idx), 1, 0, 0, rows,
                                             L.ptr(img), scale.data_ptr(), shift.data_ptr(), 0.2, classes, L.ptr(out),
                                             L.stream())


def case_gather_max():
    x = rnd(800, 32, seed=32)
    idx = torch.randint(0, 400, (2, 100, 16), generator=torch.Generator().manual_seed(33)).cuda()
    out = torch.empty(200, 32).cuda()
    return lambda: L.lib().o3dml_gather_max(L.ptr(x), 800, 32, 32, L.ptr(idx), 1, 200, 16, 100, 400, 0, L.ptr(out),
                                            32, L.stream())


def kpconv_inputs(cin, nq=200, ns=300, H=20, K=15, seed=34):
    g = torch.Generator().manual_seed(seed)
    s = torch.rand(ns, 3, generator=g).cuda()
    q = s[:nq].contiguous()
    nb = torch.randint(0, ns + 1, (nq, H), generator=g).cuda()
    x = torch.randn(ns, cin, generator=g).cuda()
    kp = ((torch.rand(K, 3, generator=g) - 0.5) * 0.3).cuda()
    off = (torch.randn(nq, 3 * K, generator=g) * 0.01).cuda()
    return q, s, nb, x, kp, off, torch.empty(nq, K * cin).cuda()


def case_kpconv_gather(cin, offset=0):
    """cin 32 / 64 / 256: grouped kernel on float4 rows, 8 / 16 / 32 lanes per query; 5: grouped kernel on narrow rows;
    10 / 50 / 130: the shuffle kernel with 1 / 2 / 4 channels per lane.  offset 4: the feature rows start 4 bytes past
    a 16-byte boundary, which the float4 kernels cannot load."""
    q, s, nb, x, kp, _, out = kpconv_inputs(cin)
    if offset:
        x = torch.cat([torch.zeros(offset // 4).cuda(), x.reshape(-1)])[offset // 4:].view_as(x)
    return lambda: L.lib().o3dml_kpconv_gather(L.ptr(q), q.shape[0], L.ptr(s), s.shape[0], L.ptr(nb), 1, nb.shape[1],
                                               L.ptr(x), cin, L.ptr(kp), kp.shape[0], 0.12, L.ptr(out), L.stream())


def case_kpconv_gather_deformable():
    q, s, nb, x, kp, off, out = kpconv_inputs(32)
    return lambda: L.lib().o3dml_kpconv_gather_deformable(L.ptr(q), q.shape[0], L.ptr(s), s.shape[0], L.ptr(nb), 1,
                                                          nb.shape[1], L.ptr(x), 32, L.ptr(kp), kp.shape[0], 0.12,
                                                          L.ptr(off), off.stride(0), L.ptr(out), L.stream())


def case_sparse_conv(cells, pre, weighted):
    """One contraction over a seeded table with shadow entries, with or without the BN-ReLU prologue, and with or
    without a weight per table entry."""
    m, n, cin, cout = 300, 250, 48, 40
    seed = 70 if weighted else 60
    g = torch.Generator().manual_seed(seed)
    table = torch.randint(0, n + n // 3, (m, cells), generator=g, dtype=torch.int32).cuda()
    weight = torch.randn(m, cells, generator=g).cuda() if weighted else None
    feat, w = rnd(n, cin, seed=seed + 1), rnd(cells, cin, cout, seed=seed + 2)
    prologue = (rnd(cin, seed=seed + 3), rnd(cin, seed=seed + 4)) if pre else None
    packed, out = LY.pack_cells(w.cpu()), torch.empty(m, cout).cuda()
    return lambda: LY.contract_cells(feat, table, packed, out, pre=prologue, entry_weight=weight)


def pv_inputs(B=2, N=500, r=6, seed=50):
    """Point rows of B clouds and their voxel coordinates and cell ids at resolution r, from o3dml_pv_voxel_cells."""
    pts = (torch.rand(B * N, 3, generator=torch.Generator().manual_seed(seed)) * 4).cuda()
    stats, vox = torch.empty(B, 4).cuda(), torch.empty(B * N, 3).cuda()
    cell = torch.empty(B * N, dtype=torch.int32).cuda()

    def call():
        return L.lib().o3dml_pv_voxel_cells(L.ptr(pts), B, N, r, 1e-6, L.ptr(stats), L.ptr(vox), L.ptr(cell),
                                            L.stream())
    return pts, vox, cell, call


def case_pv_cell_mean(B=2, N=500, r=6, C=9):
    _, _, cell, call = pv_inputs(B, N, r)
    L.check(call())
    order = torch.argsort(cell.long(), stable=True)
    ids = order.to(torch.int32)
    splits = torch.searchsorted(cell.long()[order].contiguous(), torch.arange(B * r ** 3 + 1).cuda()).contiguous()
    feat, grid = rnd(B * N, C, seed=51), torch.empty(B * r ** 3, 32).cuda()
    return lambda: L.lib().o3dml_pv_cell_mean(L.ptr(splits), L.ptr(ids), B * r ** 3, L.ptr(feat), C, C, 32,
                                              L.ptr(grid), L.stream())


def case_conv3x3x3():
    x, w = rnd(2, 5, 6, 7, 32, seed=52), rnd(27 * 32, 16, seed=53)
    weight, out = L.pack_linear(w), torch.empty(2, 5, 6, 7, 16).cuda()
    return lambda: L.conv3x3x3(x, weight, out, act="leaky", slope=0.1)


def case_trilinear_devoxelize(B=2, N=500, r=6, C=32):
    _, vox, _, call = pv_inputs(B, N, r)
    L.check(call())
    grid, out = rnd(B * r ** 3, C, seed=54), torch.zeros(B * N, C).cuda()
    inds, wgts = torch.empty(B, 8, N, dtype=torch.int32).cuda(), torch.empty(B, 8, N).cuda()
    return lambda: L.lib().o3dml_trilinear_devoxelize(L.ptr(vox), B, N, r, L.ptr(grid), C, C, 1, L.ptr(out), C,
                                                      L.ptr(inds), L.ptr(wgts), L.stream())


# ------------------------------------------------------------------------------------------------------ the tables
# {case: (the C entry the case is meant to reach, builder of its call)}.  The entries that take a workspace run over a
# workspace of exactly the size their sizing function gives.
LAUNCH_CASES = {
    "voxelize": ("o3dml_voxelize", lambda: voxelize_inputs()[2]),
    "ragged_to_dense_4B": ("o3dml_ragged_to_dense", lambda: case_ragged_to_dense(torch.int32)),
    "ragged_to_dense_8B": ("o3dml_ragged_to_dense", lambda: case_ragged_to_dense(torch.int64)),
    "knn": ("o3dml_knn_search", lambda: knn_case(p_splits=(0, 500)).with_own_workspace()),
    "knn_no_points": ("o3dml_knn_search", lambda: knn_case(p_splits=(0, 0)).with_own_workspace()),
    "knn_search_metric_ignore": ("o3dml_knn_search_metric", lambda: knn_metric_case().with_own_workspace()),
    "radius_count": ("o3dml_radius_count", lambda: radius_case().with_own_workspace()),
    "radius_fill": ("o3dml_radius_fill", lambda: after_count(radius_case())),
    "radius_search_count": ("o3dml_radius_search_count", lambda: radius_search_case().with_own_workspace()),
    "radius_search_fill": ("o3dml_radius_search_fill", lambda: after_count(radius_search_case())),
    "voxel_reduce": ("o3dml_voxel_reduce", lambda: case_voxel_reduce(False)),
    "voxel_reduce_labels": ("o3dml_voxel_reduce", lambda: case_voxel_reduce(True)),
    "reduce_subarrays_sum": ("o3dml_reduce_subarrays_sum", case_reduce_subarrays_sum),
    "sparse_conv_neighbors": ("o3dml_sparse_conv_neighbors", lambda: sparse_conv_case(200).with_own_workspace()),
    "sparse_conv_neighbors_no_inputs": ("o3dml_sparse_conv_neighbors",
                                        lambda: sparse_conv_case(0).with_own_workspace()),
    "continuous_conv": ("o3dml_continuous_conv", case_continuous_conv),
    "continuous_conv_transpose": ("o3dml_continuous_conv_transpose", case_continuous_conv_transpose),
    "invert_neighbors_list": ("o3dml_invert_neighbors_list", lambda: invert_case(5000).with_own_workspace()),
    "invert_neighbors_list_no_entries": ("o3dml_invert_neighbors_list",
                                         lambda: invert_case(0, rows=10).with_own_workspace()),
    "nms": ("o3dml_nms", lambda: nms_case(300).with_own_workspace()),
    "iou_matrix": ("o3dml_iou_matrix", case_iou_matrix),
    "pp_detect": ("o3dml_pp_detect", lambda: pp_detect_case(False).with_own_workspace()),
    "pp_detect_select": ("o3dml_pp_detect", lambda: pp_detect_case(True).with_own_workspace()),
    "pfn_scatter": ("o3dml_pp_pfn_scatter", case_pfn_scatter),
    "pfn2_scatter": ("o3dml_pp_pfn2_scatter", case_pfn2_scatter),
    "linear_simt": ("o3dml_linear", lambda: case_linear("simt")),
    "linear_tc": ("o3dml_linear_tc", lambda: case_linear("tc")),
    "linear_rows_small": ("o3dml_linear_rows_small", lambda: case_linear("rows_small")),
    "conv3x3_simt": ("o3dml_conv3x3_nhwc", lambda: case_conv3x3(False)),
    "conv3x3_tc": ("o3dml_conv3x3_nhwc_tc", lambda: case_conv3x3(True)),
    "deconv_simt": ("o3dml_deconv_nhwc", lambda: case_deconv(False)),
    "deconv_tc": ("o3dml_deconv_nhwc_tc", lambda: case_deconv(True)),
    "lfa_simt": ("o3dml_randla_lfa_pool", lambda: case_lfa("simt")),
    "lfa_tc": ("o3dml_randla_lfa_pool_tc", lambda: case_lfa("tc")),
    "lfa16": ("o3dml_randla_lfa16_pool", lambda: case_lfa("lfa16")),
    "randla_tail": ("o3dml_randla_tail", case_randla_tail),
    "gather_max": ("o3dml_gather_max", case_gather_max),
    "kpconv_gather_grouped": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(32)),
    "kpconv_gather_narrow": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(5)),
    "kpconv_gather_shuffle": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(10)),
    "kpconv_gather_grouped_16": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(64)),
    "kpconv_gather_grouped_32": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(256)),
    "kpconv_gather_shuffle_2": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(50)),
    "kpconv_gather_shuffle_4": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(130)),
    "kpconv_gather_shuffle_unaligned": ("o3dml_kpconv_gather", lambda: case_kpconv_gather(64, offset=4)),
    "kpconv_gather_deformable": ("o3dml_kpconv_gather_deformable", case_kpconv_gather_deformable),
    "sparse_conv_tc_27_pre": ("o3dml_sparse_conv_tc", lambda: case_sparse_conv(27, True, False)),
    "sparse_conv_tc_27": ("o3dml_sparse_conv_tc", lambda: case_sparse_conv(27, False, False)),
    "sparse_conv_tc_8_pre": ("o3dml_sparse_conv_tc", lambda: case_sparse_conv(8, True, False)),
    "sparse_conv_tc_1": ("o3dml_sparse_conv_tc", lambda: case_sparse_conv(1, False, False)),
    "sparse_conv_weighted_tc_27_pre": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(27, True, True)),
    "sparse_conv_weighted_tc_27": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(27, False, True)),
    "sparse_conv_weighted_tc_8_pre": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(8, True, True)),
    "sparse_conv_weighted_tc_8": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(8, False, True)),
    "sparse_conv_weighted_tc_1_pre": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(1, True, True)),
    "sparse_conv_weighted_tc_1": ("o3dml_sparse_conv_weighted_tc", lambda: case_sparse_conv(1, False, True)),
    "pv_voxel_cells": ("o3dml_pv_voxel_cells", lambda: pv_inputs()[3]),
    "pv_cell_mean": ("o3dml_pv_cell_mean", case_pv_cell_mean),
    "conv3x3x3_tc": ("o3dml_conv3x3x3_ndhwc_tc", case_conv3x3x3),
    "trilinear_devoxelize": ("o3dml_trilinear_devoxelize", case_trilinear_devoxelize),
}

# the number of kernels a case must enqueue, where the entry promises one: a sparse contraction is one launch whatever
# the number of kernel cells
EXPECTED_LAUNCHES = {case: 1 for case, (entry, _) in LAUNCH_CASES.items()
                     if entry in ("o3dml_sparse_conv_tc", "o3dml_sparse_conv_weighted_tc")}

# the kernel a case is meant to reach, for the cases that name one; with the spaces of the trace's name removed, it is
# followed by "<" or "("
EXPECTED_KERNEL = {
    **dict.fromkeys(EXPECTED_LAUNCHES, "gemm_tc_kernel"),
    "pv_voxel_cells": "pv_point_cells_kernel", "pv_cell_mean": "pv_cell_mean_kernel",
    "conv3x3x3_tc": "gemm_tc_kernel", "trilinear_devoxelize": "pv_devoxelize_kernel",
    "linear_simt": "gemm_gather_kernel", "linear_tc": "gemm_tc_kernel", "linear_rows_small": "rowmlp_kernel",
    "conv3x3_simt": "gemm_gather_kernel", "conv3x3_tc": "gemm_tc_kernel",
    "deconv_simt": "gemm_gather_kernel", "deconv_tc": "gemm_tc_kernel",
    "lfa_simt": "lfa_pool_kernel", "lfa_tc": "lfa_pool_tc_kernel", "lfa16": "lfa16c_kernel",
    "kpconv_gather_grouped": "kpconv_gather_grouped_kernel<8,4,false>",
    "kpconv_gather_narrow": "kpconv_gather_grouped_kernel<8,1,false>",
    "kpconv_gather_grouped_16": "kpconv_gather_grouped_kernel<16,4,false>",
    "kpconv_gather_grouped_32": "kpconv_gather_grouped_kernel<32,4,false>",
    "kpconv_gather_shuffle": "kpconv_gather_kernel<1>",
    "kpconv_gather_shuffle_2": "kpconv_gather_kernel<2>",
    "kpconv_gather_shuffle_4": "kpconv_gather_kernel<4>",
    "kpconv_gather_shuffle_unaligned": "kpconv_gather_kernel<2>",
    "radius_search_count": "radius_kernel<0,2,true,true>", "radius_search_fill": "radius_kernel<1,2,true,true>",
    "knn_search_metric_ignore": "knn_compact_kernel",
    "continuous_conv_transpose": "cconv_kernel<true>",
    "invert_neighbors_list": "inv_splits_kernel", "invert_neighbors_list_no_entries": "inv_splits_kernel",
    "pfn2_scatter": "pp_pfn_scatter_kernel<64,true>",
}

# {case: (the sizing function of its entries, builder)}: shapes that reach the scratch paths.
WORKSPACE_CASES = {
    "voxelize": ("o3dml_voxelize_workspace_bytes",
                 lambda: voxelize_case(splits=(0, 20000, 20000, 40000), voxel=0.1, max_voxels=30000)),
    "knn": ("o3dml_knn_workspace_bytes",
            lambda: knn_case(p_splits=(0, 3000, 3000, 6000), q_splits=(0, 2500, 5000, 5000))),
    "knn_metric_ignore": ("o3dml_knn_search_metric_workspace_bytes", knn_metric_case),
    "radius": ("o3dml_radius_workspace_bytes",
               lambda: radius_case(p_splits=(0, 3000, 3000, 6000), q_splits=(0, 2500, 5000, 5000), radius=0.3)),
    "radius_search": ("o3dml_radius_workspace_bytes", radius_search_case),
    "sparse_conv_neighbors": ("o3dml_sparse_conv_workspace_bytes", lambda: sparse_conv_case(5000)),
    "sparse_conv_neighbors_no_inputs": ("o3dml_sparse_conv_workspace_bytes", lambda: sparse_conv_case(0)),
    # 9 000 entries span five 2 048-key sort blocks; the key bound (about 3 300) takes two 8-bit passes
    "invert_neighbors_list": ("o3dml_invert_neighbors_list_workspace_bytes", lambda: invert_case(9000)),
    "invert_neighbors_list_no_entries": ("o3dml_invert_neighbors_list_workspace_bytes", lambda: invert_case(0)),
    "nms": ("o3dml_nms_workspace_bytes", lambda: nms_case(3000)),
    "pp_detect": ("o3dml_pp_detect_workspace_bytes", lambda: pp_detect_case(False)),
    "pp_detect_select": ("o3dml_pp_detect_workspace_bytes", lambda: pp_detect_case(True)),
}

# {test of tests/test_workspace.py: (the sizing function it checks, its parameter sets)}
REFUSAL_ROWS = {
    "voxelize": ("o3dml_voxelize_workspace_bytes", [(1, 1), (500, 2), (40000, 3)]),
    "knn_search": ("o3dml_knn_workspace_bytes", [(0, 1, 1), (500, 300, 1), (6000, 5000, 3)]),
    "knn_search_metric": ("o3dml_knn_search_metric_workspace_bytes",
                          [(500, 300, 1, 12, 0), (500, 300, 1, 12, 1), (6000, 5000, 3, 12, 0), (6000, 5000, 3, 12, 1)]),
    "radius_count_and_fill": ("o3dml_radius_workspace_bytes", [(1, 1, 1), (400, 200, 2), (6000, 5000, 3)]),
    "radius_search_count_and_fill": ("o3dml_radius_workspace_bytes", [(1, 1, 1), (2000, 900, 2), (6000, 5000, 3)]),
    "invert_neighbors_list": ("o3dml_invert_neighbors_list_workspace_bytes", [0, 1, 9000]),
    "nms": ("o3dml_nms_workspace_bytes", [1, 64, 65, 3000]),
    "sparse_conv_neighbors": ("o3dml_sparse_conv_workspace_bytes", [(0, 1), (1, 1), (200, 100), (5000, 100)]),
    "pp_detect": ("o3dml_pp_detect_workspace_bytes", [(1, 6, 5, 2, 3, 100), (2, 6, 5, 2, 3, 20), (1, 248, 216, 2, 3, 100),
                                                      (2, 200, 176, 4, 3, 4096)]),
}
