"""o3dml_launch_count() against the kernels the GPU actually ran.  For every C-ABI entry, on a small valid input prepared
beforehand, one call is run under torch.profiler: the counter must grow by exactly the number of kernel activities
the profiler records for that call (memsets and copies are not kernels and are not counted).  bench.py's gpu_launches
and the replay accounting of pipeline.graph_replay both rest on this counter."""
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from open3d_ml_b200 import _lib as L

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


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


# ---------------------------------------------------------------------------------------------------- the cases
# Each builder allocates everything its call needs and returns the call: a closure that only enters the library, either
# directly (returning the entry's status) or through the _lib wrapper that picks the dense kernel and checks.

def voxelize_inputs(n=500, batch=2, seed=1):
    pts = (torch.rand(n, 4, generator=torch.Generator().manual_seed(seed)) * 4).cuda()
    rs = torch.tensor([0, n // 2, n], dtype=torch.int64).cuda() if batch == 2 else torch.tensor([0, n]).cuda()
    host = [np.full(3, v, np.float32) for v in (0.5, 0.0, 4.0)]      # voxel size, range min, range max
    out = dict(coords=torch.empty(n, 3, dtype=torch.int32).cuda(), pidx=torch.empty(n, dtype=torch.int64).cuda(),
               vrs=torch.empty(n + 1, dtype=torch.int64).cuda(), bsp=torch.empty(batch + 1, dtype=torch.int64).cuda(),
               bid=torch.empty(n, dtype=torch.int32).cuda(), counts=torch.empty(2, dtype=torch.int64).cuda())
    wsb = L.lib().o3dml_voxelize_workspace_bytes(n, batch)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()

    def call():
        return L.lib().o3dml_voxelize(L.ptr(pts), n, pts.stride(0), L.ptr(rs), batch, host[0].ctypes.data,
                                      host[1].ctypes.data, host[2].ctypes.data, 32, 1000, L.ptr(out["coords"]),
                                      L.ptr(out["pidx"]), L.ptr(out["vrs"]), L.ptr(out["bsp"]), L.ptr(out["bid"]),
                                      L.ptr(out["counts"]), L.ptr(ws), wsb, L.stream())
    return pts, out, call


def case_voxelize():
    return voxelize_inputs()[2]


def case_ragged_to_dense(dtype):
    v = torch.arange(100, dtype=dtype).cuda()
    rs = torch.tensor([0, 30, 30, 100], dtype=torch.int64).cuda()
    out = torch.empty(3, 40, dtype=dtype).cuda()
    return lambda: L.lib().o3dml_ragged_to_dense(L.ptr(v), v.element_size(), 1, L.ptr(rs), 3, 40, -1, 0, L.ptr(out),
                                                 L.stream())


def case_knn(num_points):
    p, q = rnd(num_points, 3, seed=1), rnd(300, 3, seed=2)
    ps = torch.tensor([0, num_points], dtype=torch.int64).cuda()
    qs = torch.tensor([0, 300], dtype=torch.int64).cuda()
    idx, d2 = torch.empty(300, 8, dtype=torch.int32).cuda(), torch.empty(300, 8).cuda()
    wsb = L.lib().o3dml_knn_workspace_bytes(num_points, 300, 1)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()
    return lambda: L.lib().o3dml_knn_search(L.ptr(p), num_points, L.ptr(ps), L.ptr(q), 300, L.ptr(qs), 1, 8,
                                            L.ptr(idx), 0, L.ptr(d2), L.ptr(ws), wsb, L.stream())


def radius_inputs():
    p, q = rnd(400, 3, seed=3), rnd(200, 3, seed=4)
    ps = torch.tensor([0, 200, 400], dtype=torch.int64).cuda()
    qs = torch.tensor([0, 100, 200], dtype=torch.int64).cuda()
    nrs, total = torch.empty(201, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()
    wsb = L.lib().o3dml_radius_workspace_bytes(400, 200, 2)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()

    def count():
        return L.lib().o3dml_radius_count(L.ptr(p), 400, L.ptr(ps), L.ptr(q), 200, L.ptr(qs), 2, 0.8, L.ptr(nrs),
                                          L.ptr(total), L.ptr(ws), wsb, L.stream())
    return p, q, qs, nrs, total, ws, wsb, count


def case_radius_count():
    return radius_inputs()[-1]


def case_radius_fill():
    p, q, qs, nrs, total, ws, wsb, count = radius_inputs()
    L.check(count())
    t = int(total.item())
    idx, d2 = torch.empty(t, dtype=torch.int32).cuda(), torch.empty(t).cuda()
    return lambda: L.lib().o3dml_radius_fill(L.ptr(q), 400, 200, L.ptr(qs), 2, 0.8, L.ptr(nrs), L.ptr(idx), L.ptr(d2),
                                             L.ptr(ws), wsb, L.stream())


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


def case_sparse_conv_neighbors(num_in):
    ip = torch.randint(0, 8, (num_in, 3), generator=torch.Generator().manual_seed(6)).float().cuda()
    op = torch.randint(0, 8, (100, 3), generator=torch.Generator().manual_seed(7)).float().cuda()
    off, ks = np.zeros(3, np.float32), np.full(3, 3, np.int32)
    nbr, cnt = torch.empty(100, 27, dtype=torch.int32).cuda(), torch.empty(100, dtype=torch.int32).cuda()
    wsb = L.lib().o3dml_sparse_conv_workspace_bytes(num_in)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()
    return lambda: L.lib().o3dml_sparse_conv_neighbors(L.ptr(ip), num_in, L.ptr(op), 100, 1.0, off.ctypes.data,
                                                       ks.ctypes.data, 0, L.ptr(nbr), L.ptr(cnt), L.ptr(ws), wsb,
                                                       L.stream())


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


def boxes(n, seed):
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * 20
    wh = torch.rand(n, 2, generator=g) * 3 + 0.5
    return torch.cat([xy, xy + wh, torch.rand(n, 1, generator=g)], 1).cuda()


def case_nms():
    b, s = boxes(300, 12), rnd(300, seed=13)
    keep, cnt = torch.empty(300, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()
    wsb = L.lib().o3dml_nms_workspace_bytes(300)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()
    return lambda: L.lib().o3dml_nms(L.ptr(b), L.ptr(s), 300, 0.5, L.ptr(keep), L.ptr(cnt), L.ptr(ws), wsb, L.stream())


def case_iou_matrix():
    a, b = boxes(40, 14), boxes(30, 15)
    out = torch.empty(40, 30).cuda()
    return lambda: L.lib().o3dml_iou_matrix(L.ptr(a), 40, L.ptr(b), 30, 0, L.ptr(out), L.stream())


def case_pp_detect(select):
    B, H, W, A, C = 2, 6, 5, 2, 3
    nms_pre = 20 if select else 100          # select: H * W * A = 60 rows > nms_pre
    cls, reg, dr = rnd(B, A * C, H, W, seed=16), rnd(B, A * 7, H, W, seed=17) * 0.1, rnd(B, A * 2, H, W, seed=18)
    g = torch.Generator().manual_seed(19)
    anchors = torch.cat([torch.rand(H * W * A, 3, generator=g) * 20, torch.rand(H * W * A, 3, generator=g) + 1,
                         torch.rand(H * W * A, 1, generator=g)], 1).cuda()
    K = min(nms_pre, H * W * A)
    bx, sc = torch.empty(B, C * K, 7).cuda(), torch.empty(B, C * K).cuda()
    lab, cnt = torch.empty(B, C * K, dtype=torch.int64).cuda(), torch.empty(B, dtype=torch.int64).cuda()
    wsb = L.lib().o3dml_pp_detect_workspace_bytes(B, H, W, A, C, nms_pre)
    ws = torch.empty(wsb, dtype=torch.uint8).cuda()
    return lambda: L.lib().o3dml_pp_detect(L.ptr(cls), cls.stride(0), L.ptr(reg), reg.stride(0), L.ptr(dr),
                                           dr.stride(0), B, H, W, A, C, L.ptr(anchors), nms_pre, 0.1, 0.78,
                                           L.ptr(bx), L.ptr(sc), L.ptr(lab), L.ptr(cnt), L.ptr(ws), wsb, L.stream())


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


def case_kpconv_gather(cin):
    """cin 32: grouped kernel on float4 rows; 5: grouped kernel on narrow rows; 10: the shuffle kernel."""
    q, s, nb, x, kp, _, out = kpconv_inputs(cin)
    return lambda: L.lib().o3dml_kpconv_gather(L.ptr(q), q.shape[0], L.ptr(s), s.shape[0], L.ptr(nb), 1, nb.shape[1],
                                               L.ptr(x), cin, L.ptr(kp), kp.shape[0], 0.12, L.ptr(out), L.stream())


def case_kpconv_gather_deformable():
    q, s, nb, x, kp, off, out = kpconv_inputs(32)
    return lambda: L.lib().o3dml_kpconv_gather_deformable(L.ptr(q), q.shape[0], L.ptr(s), s.shape[0], L.ptr(nb), 1,
                                                          nb.shape[1], L.ptr(x), 32, L.ptr(kp), kp.shape[0], 0.12,
                                                          L.ptr(off), off.stride(0), L.ptr(out), L.stream())


CASES = {
    "voxelize": case_voxelize,
    "ragged_to_dense_4B": lambda: case_ragged_to_dense(torch.int32),
    "ragged_to_dense_8B": lambda: case_ragged_to_dense(torch.int64),
    "knn": lambda: case_knn(500),
    "knn_no_points": lambda: case_knn(0),
    "radius_count": case_radius_count,
    "radius_fill": case_radius_fill,
    "voxel_reduce": lambda: case_voxel_reduce(False),
    "voxel_reduce_labels": lambda: case_voxel_reduce(True),
    "reduce_subarrays_sum": case_reduce_subarrays_sum,
    "sparse_conv_neighbors": lambda: case_sparse_conv_neighbors(200),
    "sparse_conv_neighbors_no_inputs": lambda: case_sparse_conv_neighbors(0),
    "continuous_conv": case_continuous_conv,
    "nms": case_nms,
    "iou_matrix": case_iou_matrix,
    "pp_detect": lambda: case_pp_detect(False),
    "pp_detect_select": lambda: case_pp_detect(True),
    "pfn_scatter": case_pfn_scatter,
    "linear_simt": lambda: case_linear("simt"),
    "linear_tc": lambda: case_linear("tc"),
    "linear_rows_small": lambda: case_linear("rows_small"),
    "conv3x3_simt": lambda: case_conv3x3(False),
    "conv3x3_tc": lambda: case_conv3x3(True),
    "deconv_simt": lambda: case_deconv(False),
    "deconv_tc": lambda: case_deconv(True),
    "lfa_simt": lambda: case_lfa("simt"),
    "lfa_tc": lambda: case_lfa("tc"),
    "lfa16": lambda: case_lfa("lfa16"),
    "randla_tail": case_randla_tail,
    "gather_max": case_gather_max,
    "kpconv_gather_grouped": lambda: case_kpconv_gather(32),
    "kpconv_gather_narrow": lambda: case_kpconv_gather(5),
    "kpconv_gather_shuffle": lambda: case_kpconv_gather(10),
    "kpconv_gather_deformable": case_kpconv_gather_deformable,
}


# the kernel a case is meant to reach, where the entry chooses among several
EXPECTED_KERNEL = {
    "linear_simt": "gemm_gather_kernel", "linear_tc": "gemm_tc_kernel", "linear_rows_small": "rowmlp_kernel",
    "conv3x3_simt": "gemm_gather_kernel", "conv3x3_tc": "gemm_tc_kernel",
    "deconv_simt": "gemm_gather_kernel", "deconv_tc": "gemm_tc_kernel",
    "lfa_simt": "lfa_pool_kernel", "lfa_tc": "lfa_pool_tc_kernel", "lfa16": "lfa16c_kernel",
    "kpconv_gather_grouped": "kpconv_gather_grouped_kernel", "kpconv_gather_narrow": "kpconv_gather_grouped_kernel",
    "kpconv_gather_shuffle": "kpconv_gather_kernel",
}


@pytest.mark.parametrize("case", list(CASES))
def test_launch_count_matches_profiled_kernels(case):
    call = CASES[case]()
    torch.cuda.synchronize()
    # Every case enqueues at least one kernel.  In a long pytest process a profiling session now and then comes back
    # with no activity records at all (the CUPTI buffers of that session were not delivered); such a session says
    # nothing about the counter, so the same call is profiled again.  A trace that holds records is always compared.
    for _ in range(3):
        counted, names = counted_and_traced(call)
        if names:
            break
    assert names, "%s: no kernel activity in three profiling sessions (counter grew by %d)" % (case, counted)
    assert counted == len(names), "%s: o3dml_launch_count grew by %d, the profiler saw %d kernels: %s" % (
        case, counted, len(names), names)
    if case in EXPECTED_KERNEL:
        assert any(EXPECTED_KERNEL[case] + "<" in n or EXPECTED_KERNEL[case] + "(" in n for n in names), names
