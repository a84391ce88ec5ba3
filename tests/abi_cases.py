"""Seeded calls of the C-ABI entries that take a caller workspace, shared by tests/test_gpu_launch_count.py and
tests/test_gpu_workspace.py.  Each builder allocates the inputs and outputs of one call on the GPU and returns a WsCase
whose `run` takes the workspace as an argument, so that a test can choose where the workspace lies and how large it
is said to be.  Nothing here enters the library beyond the *_workspace_bytes sizing functions."""
import numpy as np
import torch

from open3d_ml_b200 import _lib as L


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


def boxes(n, seed):
    g = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=g) * 20
    wh = torch.rand(n, 2, generator=g) * 3 + 0.5
    return torch.cat([xy, xy + wh, torch.rand(n, 1, generator=g)], 1).cuda()


class WsCase:
    """wsb: what the entry's *_workspace_bytes returns for the case; run(ws, nbytes): the call with its workspace at
    device address ws, returning the entry's status; outputs: the tensors the call writes."""

    def __init__(self, wsb, run, outputs):
        self.wsb, self.run, self.outputs = wsb, run, outputs

    def with_own_workspace(self):
        """The call as a closure over a workspace of its own, wsb bytes."""
        ws = torch.empty(self.wsb, dtype=torch.uint8).cuda()
        return lambda: self.run(L.ptr(ws), self.wsb)


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
    case = WsCase(L.lib().o3dml_voxelize_workspace_bytes(n, batch), run, list(out.values()))
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
    return WsCase(L.lib().o3dml_knn_workspace_bytes(num_points, num_queries, batch), run, [idx, d2])


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
    case = WsCase(L.lib().o3dml_radius_workspace_bytes(num_points, num_queries, batch), count, [nrs, total])

    def prepare_fill():
        t = int(total.item())
        case.fill_outputs = [torch.zeros(t, dtype=torch.int32).cuda(), torch.zeros(t).cuda()]

    def fill(ws, nbytes):
        idx, d2 = case.fill_outputs
        return L.lib().o3dml_radius_fill(L.ptr(q), num_points, num_queries, L.ptr(qs), batch, radius, L.ptr(nrs),
                                         L.ptr(idx), L.ptr(d2), ws, nbytes, L.stream())
    case.prepare_fill, case.fill = prepare_fill, fill
    return case


def sparse_conv_case(num_in, num_out=100):
    ip = torch.randint(0, 8, (num_in, 3), generator=torch.Generator().manual_seed(6)).float().cuda()
    op = torch.randint(0, 8, (num_out, 3), generator=torch.Generator().manual_seed(7)).float().cuda()
    off, ks = np.zeros(3, np.float32), np.full(3, 3, np.int32)
    nbr, cnt = torch.empty(num_out, 27, dtype=torch.int32).cuda(), torch.empty(num_out, dtype=torch.int32).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_sparse_conv_neighbors(L.ptr(ip), num_in, L.ptr(op), num_out, 1.0, off.ctypes.data,
                                                   ks.ctypes.data, 0, L.ptr(nbr), L.ptr(cnt), ws, nbytes, L.stream())
    return WsCase(L.lib().o3dml_sparse_conv_workspace_bytes(num_in), run, [nbr, cnt])


def nms_case(n=300):
    b, s = boxes(n, 12), rnd(n, seed=13)
    keep, cnt = torch.empty(n, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_nms(L.ptr(b), L.ptr(s), n, 0.5, L.ptr(keep), L.ptr(cnt), ws, nbytes, L.stream())
    return WsCase(L.lib().o3dml_nms_workspace_bytes(n), run, [keep, cnt])


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
    return WsCase(L.lib().o3dml_pp_detect_workspace_bytes(B, H, W, A, C, nms_pre), run, [bx, sc, lab, cnt])
