"""PointPillars forward on the sm_90a kernels: the fused replacement of
``PointPillars.forward`` (ml3d/torch/models/point_pillars.py:102-134):

    voxelize (all frames in ONE batched call, no per-frame Python loop, :112-128, :328-382)
    -> pillar gather + decoration + PFN (one layer, or the two of feat_channels [64, 64]) + max + scatter-to-BEV in
       one kernel (:400-616),
       reading the CSR voxel lists directly (the [M,32,4] pillar tensor never exists)
    -> SECOND / SECONDFPN / Anchor3DHead as NHWC implicit-GEMM convolutions (:619-841)

No device->host synchronisation happens inside forward(): the voxel count stays on
the device (the reference syncs at :106 and once per frame inside the op).
The dense part (20 launches of 20-60 us each at one KITTI frame) is launch-bound from
Python, so it is captured once per canvas shape into a CUDA graph and replayed
(`use_graph=False` keeps the eager launches).
Built from a reference ``state_dict``; returns (cls, reg, dir) in NCHW like the
reference head.

Box decoding (``Anchor3DHead.get_bboxes``, :945-1025) runs on the device too: get_bboxes_padded() is one batched
call into detect.cu (top-k, decode, per-class rotated NMS) that reads nothing back to the host, and get_bboxes()
adds the one read of the per-frame counts that splitting the result into per-frame lists needs.
"""
import numpy as np
import torch

from . import _lib as L
from . import ops
from .fuse import patch
from .pipeline import BufferCache, graph_replay

BN_EPS = 1e-3  # point_pillars.py:409,648,724


class PointPillarsB200:
    """cfg keys: point_cloud_range, voxel_size, max_num_points, max_voxels (eval value),
    output_shape [ny, nx], layer_nums, layer_strides, upsample_strides; for the box decoding also
    num_classes and head = {nms_pre, score_thr, dir_offset, ranges, sizes, rotations} (cfg_from_reference)."""

    def __init__(self, state_dict, cfg, device=None, use_graph=True):
        L.require_cuda()
        self.use_graph = bool(use_graph)
        self._graphs = {}
        self.device = dev = torch.device(device or "cuda")
        self.buf = BufferCache(dev)
        self.cfg = cfg
        sd = L.host_state_dict(state_dict)
        w = self.w = {}

        def put(name, t):
            w[name] = t.to(dev, torch.float32).contiguous()

        # PFN: one layer, linear.weight [64, C+5], or two (feat_channels [64, 64]): [32, C+5] then [64, 64]
        pfn = []
        while "voxel_encoder.pfn_layers.%d.linear.weight" % len(pfn) in sd:
            pfn.append(sd["voxel_encoder.pfn_layers.%d.linear.weight" % len(pfn)])
        lw = pfn[0]
        self.point_channels = lw.shape[1] - 5
        if len(pfn) == 2 and tuple(lw.shape) == (32, lw.shape[1]) and tuple(pfn[1].shape) == (64, 64):
            self.pfn_layers = 2
        elif len(pfn) == 1:
            self.pfn_layers = 1
        else:
            raise RuntimeError("PointPillarsB200: PillarFeatureNet with linear weights %s is not fused (one layer, or "
                               "two of [32, C+5] and [64, 64])" % [list(x.shape) for x in pfn])
        self.pfn_out = pfn[-1].shape[0]
        for i, x in enumerate(pfn):
            put("pfn%d.wt" % i, x.t())
            s, t = L.fold_bn(sd, "voxel_encoder.pfn_layers.%d.norm" % i, BN_EPS)
            put("pfn%d.s" % i, s), put("pfn%d.t" % i, t)
        # backbone
        self.blocks = []
        for i, (n, stride) in enumerate(zip(cfg["layer_nums"], cfg["layer_strides"])):
            p = "backbone.blocks.%d" % i
            layers = [(p + ".0", p + ".1", stride)]
            layers += [("%s.%d" % (p, 3 + 3 * j), "%s.%d" % (p, 4 + 3 * j), 1) for j in range(n)]
            for conv, bn, st in layers:
                cw = sd[conv + ".weight"]  # [co, ci, 3, 3]
                w[conv + ".wt"] = L.pack_linear(cw.permute(2, 3, 1, 0).reshape(9 * cw.shape[1], cw.shape[0]))
                s, t = L.fold_bn(sd, bn, BN_EPS)
                put(conv + ".s", s), put(conv + ".t", t)
            self.blocks.append([(c, st, sd[c + ".weight"].shape[1], sd[c + ".weight"].shape[0])
                                for c, _, st in layers])
        # neck
        self.deblocks = []
        for i, us in enumerate(cfg["upsample_strides"]):
            p = "neck.deblocks.%d" % i
            dw = sd[p + ".0.weight"]  # ConvTranspose2d [ci, co, k, k]
            if dw.shape[2] != us or dw.shape[3] != us:
                raise RuntimeError("PointPillarsB200: deblock kernel must equal its stride")
            co = dw.shape[1]
            w[p + ".wt"] = L.pack_linear(dw.permute(0, 2, 3, 1).reshape(dw.shape[0], us * us * co))
            s, t = L.fold_bn(sd, p + ".1", BN_EPS)
            put(p + ".s", s.repeat(us * us)), put(p + ".t", t.repeat(us * us))
            self.deblocks.append((p, us, dw.shape[0], co))
        self.neck_channels = sum(d[3] for d in self.deblocks)
        # head: three 1x1 convs as one GEMM
        hw = [sd["bbox_head.%s.weight" % h][:, :, 0, 0] for h in ("conv_cls", "conv_reg", "conv_dir_cls")]
        hb = [sd["bbox_head.%s.bias" % h] for h in ("conv_cls", "conv_reg", "conv_dir_cls")]
        self.head_split = [x.shape[0] for x in hw]
        w["head.wt"] = L.pack_linear(torch.cat(hw, 0).t())
        put("head.t", torch.cat(hb, 0))
        r = cfg["point_cloud_range"]
        self.vx, self.vy = float(cfg["voxel_size"][0]), float(cfg["voxel_size"][1])
        # same float64->float32 path as PillarFeatureNet.__init__ (:506-509)
        self.x_off = float(self.vx / 2 + r[0])
        self.y_off = float(self.vy / 2 + r[1])
        self.ny, self.nx = cfg["output_shape"]
        self._anchors = {}

    # ------------------------------------------------------------- front end
    def front_end(self, frames, want_feat=False, canvas_nchw=False):
        """frames: list of [N_i, C] float32 tensors (CPU or CUDA).  Returns the zero-initialised
        canvas with the pillar features scattered, plus the raw voxel buffers."""
        cfg, dev = self.cfg, self.device
        B = len(frames)
        pts = torch.cat([f.to(dev, non_blocking=True) for f in frames], 0).contiguous()
        lens = [0] + [int(f.shape[0]) for f in frames]
        rs = torch.tensor(np.cumsum(lens), dtype=torch.int64).to(dev, non_blocking=True)
        r = cfg["point_cloud_range"]
        coords, pidx, vrs, bsp, bid, counts = ops.voxelize_raw(
            pts[:, :3], rs, cfg["voxel_size"], r[:3], r[3:], cfg["max_num_points"],
            cfg["max_voxels"], want_batch_id=True)
        C = self.pfn_out
        shape = (B, C, self.ny, self.nx) if canvas_nchw else (B, self.ny, self.nx, C)
        canvas = self.buf.get("canvas", shape)
        canvas.zero_()
        bound = min(pts.shape[0], B * int(cfg["max_voxels"]))
        feat = torch.empty((bound, C), dtype=torch.float32, device=dev) if want_feat else None
        vox = dict(coords=coords, point_indices=pidx, row_splits=vrs, batch_splits=bsp, batch_id=bid, counts=counts,
                   feat=feat, points=pts, bound=bound)
        self.pfn_scatter(vox, canvas, canvas_nchw)
        return canvas, vox

    def pfn_scatter(self, vox, canvas, canvas_nchw=False):
        """The pillar feature net + scatter of front_end (one launch): the voxel buffers `vox` of front_end into
        vox["feat"] (may be None) and `canvas`."""
        w = self.w
        voxels = (L.ptr(vox["points"]), vox["points"].stride(0), self.point_channels, L.ptr(vox["coords"]),
                  L.ptr(vox["row_splits"]), L.ptr(vox["point_indices"]), L.ptr(vox["batch_id"]), L.ptr(vox["counts"]),
                  vox["bound"], L.ptr(w["pfn0.wt"]), L.ptr(w["pfn0.s"]), L.ptr(w["pfn0.t"]))
        rest = (self.pfn_out, self.vx, self.vy, self.x_off, self.y_off, self.nx, self.ny,
                int(self.cfg["max_num_points"]), L.ptr(vox["feat"]), L.ptr(canvas), 1 if canvas_nchw else 0, L.stream())
        if self.pfn_layers == 2:
            L.check(L.lib().o3dml_pp_pfn2_scatter(*voxels, L.ptr(w["pfn1.wt"]), L.ptr(w["pfn1.s"]),
                                                  L.ptr(w["pfn1.t"]), *rest))
        else:
            L.check(L.lib().o3dml_pp_pfn_scatter(*voxels, *rest))

    # ---------------------------------------------------------- dense layers
    def _conv(self, x, B, H, W, name, stride, cin, cout):
        OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
        out = self.buf.get(name, (B, OH, OW, cout))
        L.conv3x3(x, self.w[name + ".wt"], out, self.w[name + ".s"], self.w[name + ".t"], stride, act="relu")
        return out, OH, OW

    def backbone_neck_head(self, canvas):
        """SECOND + SECONDFPN + Anchor3DHead on the NHWC canvas -> (cls, reg, dir) in NCHW."""
        if not self.use_graph:
            return self._bnh_eager(canvas)
        return graph_replay(self._graphs, "backbone_neck_head", [canvas], lambda: self._bnh_eager(canvas), self.device)

    def _bnh_eager(self, canvas):
        B, H, W = canvas.shape[0], canvas.shape[1], canvas.shape[2]
        x = canvas
        feats = []
        for layers in self.blocks:
            for name, stride, cin, cout in layers:
                x, H, W = self._conv(x, B, H, W, name, stride, cin, cout)
            feats.append((x, H, W))
        us0 = self.deblocks[0][1]
        OH, OW = feats[0][1] * us0, feats[0][2] * us0
        neck = self.buf.get("neck", (B, OH, OW, self.neck_channels))
        off = 0
        for (p, us, cin, co), (f, h, w_) in zip(self.deblocks, feats):
            if h * us != OH or w_ * us != OW:
                raise RuntimeError("PointPillarsB200: neck scales do not line up")
            L.deconv(f, self.w[p + ".wt"], neck[..., off:off + co], self.w[p + ".s"], self.w[p + ".t"], us,
                     act="relu")
            off += co
        ch = sum(self.head_split)
        out = torch.empty((B, ch, OH, OW), dtype=torch.float32, device=self.device)
        L.linear([L.make_src(neck.view(B * OH * OW, self.neck_channels))], self.w["head.wt"], out,
                 None, self.w["head.t"], act=None, num_rows=B * OH * OW, out_channels=ch,
                 out_nchw_plane=OH * OW)
        a, b_, _ = self.head_split
        return out[:, :a], out[:, a:a + b_], out[:, a + b_:]

    def forward(self, frames):
        if hasattr(frames, "point"):
            frames = frames.point
        canvas, _ = self.front_end(frames)
        return self.backbone_neck_head(canvas)

    __call__ = forward

    # ---------------------------------------------------------- box decoding
    def _head_cfg(self):
        head, nc = self.cfg.get("head"), self.cfg.get("num_classes")
        if head is None or nc is None:
            raise RuntimeError("PointPillarsB200: box decoding needs cfg['head'] and cfg['num_classes'] "
                               "(cfg_from_reference builds both)")
        A = len(head["sizes"]) * len(head["rotations"])
        if self.head_split != [A * nc, A * 7, A * 2]:
            raise RuntimeError("PointPillarsB200: head channels %s do not match %d anchors x %d classes"
                               % (self.head_split, A, nc))
        return head, int(nc), A

    def anchors(self, H, W, device):
        """Anchor3DRangeGenerator.grid_anchors (objdet_helper.py:164-245) as [H * W * A, 7], row (y * W + x) * A + a,
        a = size * R + rotation; built once per (H, W, device) with torch.linspace on that device, as the reference
        builds it (torch's CPU and CUDA linspace round differently, so it is not recomputed in a kernel)."""
        head, _, _ = self._head_cfg()
        key = (int(H), int(W), str(device))
        t = self._anchors.get(key)
        if t is None:
            t = self._anchors[key] = grid_anchors(head, H, W, device)
        return t

    def get_bboxes_padded(self, cls, reg, dir):
        """Head maps of B frames (NCHW, any batch stride) -> (boxes [B, C*K, 7], scores [B, C*K], labels int64 [B, C*K],
        counts int64 [B]) with K = min(nms_pre, H * W * A).  Frame b's boxes are rows [0, counts[b]): class 0's in
        NMS visiting order, then class 1's, ...; the rows after them are zero with label -1.  No host synchronisation;
        capturable into a CUDA graph (DESIGN.md section 2, "PointPillars box decoding")."""
        head, C, A = self._head_cfg()
        B, _, H, W = cls.shape
        maps = []
        for t, ch in ((cls, A * C), (reg, A * 7), (dir, A * 2)):
            if t.dim() != 4 or tuple(t.shape) != (B, ch, H, W):
                raise RuntimeError("PointPillarsB200.get_bboxes: map of shape %s, expected %s"
                                   % (tuple(t.shape), (B, ch, H, W)))
            if t.dtype != torch.float32 or not t.is_cuda:
                raise RuntimeError("PointPillarsB200.get_bboxes: maps must be float32 CUDA tensors")
            if t.stride(3) != 1 or t.stride(2) != W or t.stride(1) != H * W:
                t = t.contiguous()
            maps.append(t)
        nms_pre = int(head["nms_pre"])
        lib = L.lib()
        ws_bytes = lib.o3dml_pp_detect_workspace_bytes(B, H, W, A, C, nms_pre)
        if ws_bytes == 0:
            L.check(lib.o3dml_pp_detect(None, 0, None, 0, None, 0, B, H, W, A, C, None, nms_pre, 0.0, 0.0,
                                        None, None, None, None, None, 0, L.stream()))
        K = min(nms_pre, H * W * A)
        dev = cls.device
        boxes = torch.empty((B, C * K, 7), dtype=torch.float32, device=dev)
        scores = torch.empty((B, C * K), dtype=torch.float32, device=dev)
        labels = torch.empty((B, C * K), dtype=torch.int64, device=dev)
        counts = torch.empty((B,), dtype=torch.int64, device=dev)
        ws = L.workspace(ws_bytes, dev)
        anchors = self.anchors(H, W, dev)
        c, r, d = maps
        L.check(lib.o3dml_pp_detect(L.ptr(c), c.stride(0), L.ptr(r), r.stride(0), L.ptr(d), d.stride(0), B, H, W, A, C,
                                    L.ptr(anchors), nms_pre, float(head["score_thr"]), float(head["dir_offset"]),
                                    L.ptr(boxes), L.ptr(scores), L.ptr(labels), L.ptr(counts), L.ptr(ws), ws_bytes,
                                    L.stream()))
        return boxes, scores, labels, counts

    def get_bboxes(self, cls, reg, dir):
        """Anchor3DHead.get_bboxes: (list of boxes [n_b, 7], list of scores [n_b], list of labels int64 [n_b]) per
        frame, all on the device.  One device-to-host read (the per-frame counts)."""
        boxes, scores, labels, counts = self.get_bboxes_padded(cls, reg, dir)
        n = counts.tolist()
        return ([boxes[b, :k] for b, k in enumerate(n)], [scores[b, :k] for b, k in enumerate(n)],
                [labels[b, :k] for b, k in enumerate(n)])


def grid_anchors(head, H, W, device):
    """The anchors of a head cfg for an H x W map as [H * W * A, 7] (see PointPillarsB200.anchors)."""
    sizes = torch.tensor(head["sizes"], device=device).reshape(-1, 3)
    ranges = list(head["ranges"])
    if len(ranges) != len(sizes):
        ranges = ranges * len(sizes)
    rots = torch.tensor(head["rotations"], device=device)
    S, R = sizes.shape[0], rots.shape[0]
    t = torch.empty((H, W, S, R, 7), dtype=torch.float32, device=device)
    for s in range(S):
        # the float32 range values, as the reference's torch.tensor(anchor_range); host floats, so that building
        # the anchors reads nothing back from the device
        r = torch.tensor(ranges[s], dtype=torch.float32).tolist()
        t[:, :, s, :, 0] = torch.linspace(r[0], r[3], W, device=device).view(1, W, 1)
        t[:, :, s, :, 1] = torch.linspace(r[1], r[4], H, device=device).view(H, 1, 1)
        t[:, :, s, :, 2] = torch.linspace(r[2], r[5], 1, device=device)
        t[:, :, s, :, 3:6] = sizes[s]
        t[:, :, s, :, 6] = rots
    return t.view(H * W * S * R, 7)


def _head_from_reference(head, classes):
    """Anchor3DHead's decoding parameters with its constructor defaults (point_pillars.py:760-770)."""
    head = head or {}
    return dict(nms_pre=int(head.get("nms_pre", 100)), score_thr=float(head.get("score_thr", 0.1)),
                dir_offset=float(head.get("dir_offset", 0)),
                ranges=[list(map(float, r)) for r in head.get("ranges", [[0, -40.0, -3, 70.0, 40.0, 1]])],
                sizes=[list(map(float, s)) for s in head.get("sizes", [[0.6, 1.0, 1.5]])],
                rotations=[float(r) for r in head.get("rotations", [0, 1.57])]), len(classes)


def cfg_from_reference(model_cfg):
    """Builds the cfg dict from a reference yml `model:` section (pointpillars_kitti.yml:7-66)."""
    head, num_classes = _head_from_reference(model_cfg.get("head"), model_cfg.get("classes", ["car"]))
    return dict(point_cloud_range=list(model_cfg["point_cloud_range"]),
                voxel_size=list(model_cfg["voxelize"]["voxel_size"]),
                max_num_points=model_cfg["voxelize"]["max_num_points"],
                max_voxels=model_cfg["voxelize"]["max_voxels"][1],
                output_shape=list(model_cfg["scatter"]["output_shape"]),
                layer_nums=list(model_cfg["backbone"]["layer_nums"]),
                layer_strides=list(model_cfg["backbone"]["layer_strides"]),
                upsample_strides=list(model_cfg["neck"]["upsample_strides"]),
                head=head, num_classes=num_classes)


def fused_from_reference(model):
    """The fused model of a reference ``PointPillars`` instance, from its current ``state_dict()`` and the
    modules' own attributes."""
    vl, hd = model.voxel_layer, model.bbox_head
    gen = hd.anchor_generator
    cfg = dict(point_cloud_range=list(model.point_cloud_range), voxel_size=[float(v) for v in vl.voxel_size],
               max_num_points=int(vl.max_num_points), max_voxels=int(vl.max_voxels[1]),
               output_shape=[int(model.middle_encoder.ny), int(model.middle_encoder.nx)],
               layer_nums=[(len(blk) - 3) // 3 for blk in model.backbone.blocks],
               layer_strides=[int(blk[0].stride[0]) for blk in model.backbone.blocks],
               upsample_strides=[int(d[0].stride[0]) for d in model.neck.deblocks],
               head=dict(nms_pre=int(hd.nms_pre), score_thr=float(hd.score_thr), dir_offset=float(hd.dir_offset),
                         ranges=[[float(v) for v in r] for r in gen.ranges],
                         sizes=[[float(v) for v in s] for s in gen.sizes],
                         rotations=[float(r) for r in gen.rotations]),
               num_classes=int(hd.num_classes))
    return PointPillarsB200(model.state_dict(), cfg)


def patch_reference_model(model):
    """Makes a reference ``PointPillars`` instance forward and decode boxes on the fused path (see ``fuse.patch``)."""
    return patch(model, fused_from_reference)
