"""PVCNN forward on the sm_90a kernels: the fused replacement of ``PVCNN.forward``
(ml3d/torch/models/pvcnn.py:136-160) and of the layers it calls (PVConv :559-576, Voxelization :642-664,
avg_voxelize :579-619, SharedMLP :455-501, the cloud and classifier MLPs :358-408).

The module is built from a reference ``state_dict``, folds the eval-mode BatchNorms (eps 1e-4 for the BatchNorm3d of
the voxel branch, 1e-5 for every BatchNorm1d) and keeps every activation as point rows [B*N, C] or as a
channels-last grid [B, X, Y, Z, C].  Per PVConv block:

    cell_mean(points grouped by cell) -> conv3x3x3 -> conv3x3x3           (voxel branch, tensor cores)
    linear(point branch) -> the block's column slice of the concat buffer
    trilinear_devoxelize(accumulate) adds the voxel branch onto that slice

The points are grouped by cell once per distinct resolution (o3dml_invert_neighbors_list over one cell id per point is
the stable counting sort).  The five block outputs share one [B*N, 1344] buffer, the classifier's single source; the
broadcast cloud feature enters the first classifier layer as a per-cloud shift vector and is never materialised.
Inference only; no host read anywhere in the forward.
"""
import torch

from . import _lib as L
from .fuse import patch
from .pipeline import BufferCache, graph_replay

BN3D_EPS = 1e-4      # pvcnn.py:544,551
BN1D_EPS = 1e-5      # torch default: SharedMLP :470, _linear_bn_relu :355
VOXEL_EPS = 1e-6     # create_pointnet_components :415
LEAKY = 0.1          # pvcnn.py:545,552
BLOCKS = ((64, 1, 32), (64, 2, 16), (128, 1, 16))   # PVCNN.blocks[:-1]: (channels, repeats, resolution)
MAX_K = 64           # points per row of the first level of the max over a cloud


def pad32(c):
    return (c + 31) // 32 * 32


def cfg_from_reference(cfg):
    """The reference's model section (pvcnn_s3dis.yml) -> the keys PVCNNB200 reads."""
    return dict(num_classes=int(cfg.get("num_classes", 13)),
                extra_feature_channels=int(cfg.get("extra_feature_channels", 6)),
                width_multiplier=cfg.get("width_multiplier", 1),
                voxel_resolution_multiplier=cfg.get("voxel_resolution_multiplier", 1))


def block_resolutions(cfg):
    vr = cfg.get("voxel_resolution_multiplier", 1)
    return [int(vr * res) for _, rep, res in BLOCKS for _ in range(rep)]


class PVCNNB200:
    def __init__(self, state_dict, cfg, device=None, use_graph=True):
        L.require_cuda()
        if cfg.get("with_se", False):
            raise RuntimeError("PVCNNB200: with_se=True (SE3d) is not built; PVCNN never constructs it")
        self.device = torch.device(device or "cuda")
        self.use_graph = bool(use_graph)
        self._graphs = {}
        self._consts = {}
        self.buf = BufferCache(self.device)
        self.res = block_resolutions(cfg)
        self.in_channels = int(cfg.get("extra_feature_channels", 6)) + 3
        sd = L.host_state_dict(state_dict)
        if any(".voxel_layers.6." in k for k in sd):
            raise RuntimeError("PVCNNB200: the state_dict holds SE3d layers (with_se=True), which are not built")
        nb = len(self.res)
        w0 = sd["point_features.0.point_features.layers.0.weight"]
        if w0.shape[1] != self.in_channels:
            raise RuntimeError("PVCNNB200: the state_dict takes %d input channels, the config says %d"
                               % (w0.shape[1], self.in_channels))
        self.w = {}
        dev = self.device

        def put(name, t):
            self.w[name] = t.to(dev, torch.float32).contiguous()

        def dense(name, w_out_in, bn, bias, eps=BN1D_EPS):
            self.w[name + ".wt"] = L.pack_linear(w_out_in.t())
            if bn is None:
                put(name + ".t", bias)
            else:
                s, t = L.fold_bn(sd, bn, eps, bias)
                put(name + ".s", s), put(name + ".t", t)

        self.widths = []
        for i in range(nb):
            p = "point_features.%d" % i
            for j, li in enumerate((0, 3)):
                w = sd["%s.voxel_layers.%d.weight" % (p, li)]           # [Cout, Cin, kx, ky, kz]
                co, ci = w.shape[:2]
                wp = torch.zeros((27, pad32(ci), co))
                wp[:, :ci] = w.permute(2, 3, 4, 1, 0).reshape(27, ci, co)
                self.w["%s.conv%d.wt" % (p, j)] = L.pack_linear(wp.reshape(27 * pad32(ci), co))
                s, t = L.fold_bn(sd, "%s.voxel_layers.%d" % (p, li + 1), BN3D_EPS,
                                 sd["%s.voxel_layers.%d.bias" % (p, li)])
                put("%s.conv%d.s" % (p, j), s), put("%s.conv%d.t" % (p, j), t)
            dense(p + ".point", sd[p + ".point_features.layers.0.weight"][:, :, 0],
                  p + ".point_features.layers.1", sd[p + ".point_features.layers.0.bias"])
            self.widths.append(co)
            if co % 32:
                raise RuntimeError("PVCNNB200: block %d is %d channels wide; the voxel convolutions take multiples of 32"
                                   % (i, co))
        p = "point_features.%d" % nb
        dense(p, sd[p + ".layers.0.weight"][:, :, 0], p + ".layers.1", sd[p + ".layers.0.bias"])
        self.widths.append(sd[p + ".layers.0.weight"].shape[0])
        self.ccat = sum(self.widths)
        for j in (0, 1):
            p = "cloud_features.%d" % j
            dense(p, sd[p + ".0.weight"], p + ".1", sd[p + ".0.bias"])
        # classifier.0 over [concat | cloud feature]: the concat rows are the layer's weight, the cloud-feature rows
        # become a [cloud channels, 512] product whose result, scaled and shifted by the folded BN, is the per-cloud shift
        w1 = sd["classifier.0.layers.0.weight"][:, :, 0]
        dense("classifier.0", w1[:, :self.ccat], "classifier.0.layers.1", sd["classifier.0.layers.0.bias"])
        self.w["classifier.0.cloud.wt"] = L.pack_linear(w1[:, self.ccat:].t())
        dense("classifier.2", sd["classifier.2.layers.0.weight"][:, :, 0], "classifier.2.layers.1",
              sd["classifier.2.layers.0.bias"])
        dense("classifier.4", sd["classifier.4.weight"][:, :, 0], None, sd["classifier.4.bias"])
        self.num_classes = sd["classifier.4.weight"].shape[0]

    def _lin(self, name, srcs, out, act="relu", shift=None, **kw):
        return L.linear(srcs, self.w[name + ".wt"], out, self.w.get(name + ".s"),
                        self.w[name + ".t"] if shift is None else shift, act=act, **kw)

    def _const(self, key, make):
        t = self._consts.get(key)
        if t is None:
            t = self._consts[key] = make()
        return t

    # ------------------------------------------------------------------ steps
    def voxel_cells(self, coords, B, N, r):
        """coords [B*N, 3] -> (voxel coordinates [B*N, 3], cell row splits [B r^3 + 1], point ids by cell [B*N])."""
        tag = "r%d." % r
        vox = self.buf.get(tag + "vox", (B * N, 3))
        cell = self.buf.get(tag + "cell", (B * N,), torch.int32)
        stats = self.buf.get(tag + "stats", (B, 4))
        L.check(L.lib().o3dml_pv_voxel_cells(L.ptr(coords), B, N, r, VOXEL_EPS, L.ptr(stats), L.ptr(vox), L.ptr(cell),
                                             L.stream()))
        cells = B * r ** 3
        ids = self.buf.get(tag + "ids", (B * N,), torch.int32)
        splits = self.buf.get(tag + "splits", (cells + 1,), torch.int64)
        perm = self.buf.get("perm", (B * N,), torch.int64)
        iota = self._const(("iota", B * N), lambda: torch.arange(B * N + 1, dtype=torch.int64, device=self.device))
        wsb = L.lib().o3dml_invert_neighbors_list_workspace_bytes(B * N)
        ws = self.buf.get("invert.ws", (wsb,), torch.uint8)
        L.check(L.lib().o3dml_invert_neighbors_list(cells, L.ptr(cell), 0, L.ptr(iota), B * N, B * N, L.ptr(ids),
                                                    L.ptr(splits), L.ptr(perm), L.ptr(ws), wsb, L.stream()))
        return vox, splits, ids

    def cloud_max(self, x, B, N):
        """max over the N rows of each cloud of x [B*N, C] -> [B, C]: two levels of gather_max over constant ids."""
        C = x.shape[1]
        k1 = min(MAX_K, N)
        n1 = (N + k1 - 1) // k1

        def level1():
            j = torch.arange(n1 * k1, device=self.device).clamp(max=N - 1).view(1, n1, k1)
            return (j + torch.arange(B, device=self.device).view(B, 1, 1) * N).to(torch.int32).contiguous()

        def level2():
            return torch.arange(B * n1, dtype=torch.int32, device=self.device).view(B, n1).contiguous()
        i1, i2 = self._const(("max1", B, N), level1), self._const(("max2", B, N), level2)
        part = self.buf.get("max.part", (B * n1, C))
        out = self.buf.get("max.out", (B, C))
        L.check(L.lib().o3dml_gather_max(L.ptr(x), B * N, C, x.stride(0), L.ptr(i1), 0, B * n1, k1, 0, 0, 0,
                                         L.ptr(part), C, L.stream()))
        L.check(L.lib().o3dml_gather_max(L.ptr(part), B * n1, C, C, L.ptr(i2), 0, B, n1, 0, 0, 0, L.ptr(out), C,
                                         L.stream()))
        return out

    # ------------------------------------------------------------------ forward
    def forward(self, inputs, taps=None):
        dev = self.device
        point, feat = inputs["point"].to(dev, non_blocking=True), inputs["feat"].to(dev, non_blocking=True)
        B, _, N = point.shape
        if feat.shape[1] != self.in_channels:
            raise RuntimeError("PVCNNB200: feat has %d channels, the model takes %d" % (feat.shape[1], self.in_channels))
        coords = self.buf.get("coords", (B * N, 3))
        coords.view(B, N, 3).copy_(point.permute(0, 2, 1))
        x = self.buf.get("feat", (B * N, self.in_channels))
        x.view(B, N, -1).copy_(feat.permute(0, 2, 1))
        cat = self.buf.get("cat", (B * N, self.ccat))
        groups = {}
        off = 0
        for i, r in enumerate(self.res):
            p = "point_features.%d" % i
            if r not in groups:
                groups[r] = self.voxel_cells(coords, B, N, r)
            vox, splits, ids = groups[r]
            cin, co = x.shape[1], self.widths[i]
            cells = B * r ** 3
            g0 = self.buf.get("grid.in.%d.%d" % (r, pad32(cin)), (B, r, r, r, pad32(cin)))
            L.check(L.lib().o3dml_pv_cell_mean(L.ptr(splits), L.ptr(ids), cells, L.ptr(x), x.stride(0), cin,
                                               pad32(cin), L.ptr(g0), L.stream()))
            g1 = self.buf.get("grid.a.%d.%d" % (r, co), (B, r, r, r, co))
            g2 = self.buf.get("grid.b.%d.%d" % (r, co), (B, r, r, r, co))
            L.conv3x3x3(g0, self.w[p + ".conv0.wt"], g1, self.w[p + ".conv0.s"], self.w[p + ".conv0.t"], "leaky", LEAKY)
            L.conv3x3x3(g1, self.w[p + ".conv1.wt"], g2, self.w[p + ".conv1.s"], self.w[p + ".conv1.t"], "leaky", LEAKY)
            y = cat[:, off:off + co]
            self._lin(p + ".point", [L.make_src(x)], y)
            L.check(L.lib().o3dml_trilinear_devoxelize(L.ptr(vox), B, N, r, L.ptr(g2), co, co, 1, L.ptr(y), self.ccat,
                                                       None, None, L.stream()))
            if taps is not None:
                # copies: blocks of one resolution and width share their grids
                taps[p + ".voxels"] = g0[..., :cin].permute(0, 4, 1, 2, 3).clone()
                taps[p + ".conv0"] = g1.permute(0, 4, 1, 2, 3).clone()
                taps[p + ".conv1"] = g2.permute(0, 4, 1, 2, 3).clone()
                taps[p] = y.reshape(B, N, co).clone()
            x, off = y, off + co
        y = cat[:, off:]
        self._lin("point_features.%d" % len(self.res), [L.make_src(x)], y)
        cf = self.cloud_max(y, B, N)
        for j in (0, 1):
            p = "cloud_features.%d" % j
            cf = self._lin(p, [L.make_src(cf)], self.buf.get(p, (B, self.w[p + ".wt"].shape[1])))
        if taps is not None:
            taps["cloud_features"] = cf.clone()
        c1 = self.w["classifier.0.wt"].shape[1]
        shift = self.buf.get("classifier.0.shift", (B, c1))
        L.linear([L.make_src(cf)], self.w["classifier.0.cloud.wt"], shift, self.w["classifier.0.s"],
                 self.w["classifier.0.t"])
        h1 = self.buf.get("classifier.0", (B * N, c1))
        for b in range(B):
            rows = slice(b * N, (b + 1) * N)
            self._lin("classifier.0", [L.make_src(cat[rows])], h1[rows], shift=shift[b])
        h2 = self._lin("classifier.2", [L.make_src(h1)],
                       self.buf.get("classifier.2", (B * N, self.w["classifier.2.wt"].shape[1])))
        logits = torch.empty((B * N, self.num_classes), dtype=torch.float32, device=dev)
        self._lin("classifier.4", [L.make_src(h2)], logits, act=None)
        return logits.view(B, N, self.num_classes)

    __call__ = forward

    def forward_graphed(self, inputs):
        """forward() for DEVICE-resident inputs, replayed from a CUDA graph keyed by their addresses."""
        flat = [inputs["point"], inputs["feat"]]
        if not self.use_graph or not all(t.is_cuda for t in flat):
            return self.forward(inputs)
        return graph_replay(self._graphs, "forward", flat, lambda: self.forward(inputs), self.device)


def fused_from_reference(model):
    """The fused model of a reference ``PVCNN`` instance, from its current ``state_dict()`` and ``cfg``."""
    return PVCNNB200(model.state_dict(), cfg_from_reference(model.cfg))


def patch_reference_model(model):
    """Makes a reference ``PVCNN`` instance run its forward on the fused path (see ``fuse.patch``)."""
    return patch(model, fused_from_reference)
