"""KPFCNN forward on the sm_90a kernels: the fused replacement of ``KPFCNN.forward``
(ml3d/torch/models/kpconv.py:270-291) for rigid and deformable (modulated = False) KPConv with
linear influence and sum aggregation: every shipped config, Paris-Lille3D's deformable layers
included (SURVEY.md A11).

  KPConv.forward (:1005-1159)  = kpconv_gather (neighbour gather + kernel-point influence,
                                  one group of lanes per query) + gathered GEMM [15*Cin, Cout]
                                  with BN + LeakyReLU in the epilogue
  deformable KPConv (:1011-1106) = rigid kpconv_gather + GEMM [15*Cin, 45] + offset_bias (the
                                  offset conv), then kpconv_gather_deformable (per-query kernel
                                  points, out-of-range neighbours dropped), then the same GEMM;
                                  the kernel points are KPConv.offset_conv.kernel_points (DESIGN §2)
  UnaryBlock (:1255-1295)       = gathered GEMM (+ residual + LeakyReLU for the resnet tail)
  max_pool / closest_pool (:821-858) = gather_max / index operand of the GEMM
  decoder concat (:283-285)     = two-source GEMM, nothing is materialised

Built from a reference ``state_dict`` (kernel points travel in it, SURVEY.md A8) plus the
architecture list; the batch object is the reference's (points / neighbors / pools /
upsamples / features), CPU or CUDA, int64 or int32 indices.  ``patch_reference_model`` puts it
behind a reference ``KPFCNN`` instance's forward.
"""
import torch

from . import _lib as L

BN_EPS = 1e-5  # nn.BatchNorm1d default, kpconv.py:1231


def _plan(cfg):
    """Mirrors KPFCNN.__init__ (kpconv.py:128-249)."""
    arch = cfg["architecture"]
    r = cfg["first_subsampling_dl"] * cfg["conv_radius"]
    in_dim, out_dim, layer = cfg["in_features_dim"], cfg["first_features_dim"], 0
    enc, skips, skip_dims = [], [], []
    for bi, blk in enumerate(arch):
        if any(t in blk for t in ("pool", "strided", "upsample", "global")):
            skips.append(bi)
            skip_dims.append(in_dim)
        if "upsample" in blk:
            break
        if not ("simple" in blk or "resnetb" in blk):
            raise RuntimeError("KPFCNNB200: block '%s' is not supported by the fused path" % blk)
        enc.append(dict(kind=blk, in_dim=in_dim, out_dim=out_dim, layer=layer, deform="deform" in blk,
                        extent=r * cfg["KP_extent"] / cfg["conv_radius"]))
        in_dim = out_dim // 2 if "simple" in blk else out_dim
        if "pool" in blk or "strided" in blk:
            layer += 1
            r *= 2
            out_dim *= 2
    start = next(i for i, b in enumerate(arch) if "upsample" in b)
    dec, concats = [], []
    for bi, blk in enumerate(arch[start:]):
        if bi > 0 and "upsample" in arch[start + bi - 1]:
            in_dim += skip_dims[layer]
            concats.append(bi)
        dec.append(dict(kind=blk, in_dim=in_dim, out_dim=out_dim, layer=layer))
        in_dim = out_dim
        if bi == 0 and cfg.get("reduce_fc", False):       # kpconv.py:219-220
            out_dim //= 2
        if "upsample" in blk:
            layer -= 1
            r *= 0.5
            out_dim //= 2
    return enc, skips, dec, concats


class KPFCNNB200:
    def __init__(self, state_dict, cfg, device=None):
        L.require_cuda()
        self.device = dev = torch.device(device or "cuda")
        self.cfg = cfg
        if cfg.get("KP_influence", "linear") != "linear" or cfg.get("aggregation_mode", "sum") != "sum":
            raise RuntimeError("KPFCNNB200: only KP_influence=linear, aggregation_mode=sum")
        self.slope = float(cfg.get("l_relu", 0.1))
        self.use_bn = bool(cfg.get("use_batch_norm", True))
        self.enc, self.enc_skips, self.dec, self.dec_concats = _plan(cfg)
        if cfg.get("modulated", False) and any(b["deform"] for b in self.enc):
            raise RuntimeError("KPFCNNB200: modulated deformable KPConv is not supported")
        sd = L.host_state_dict(state_dict)
        w = self.w = {}

        def put(name, t):
            w[name] = t.to(dev, torch.float32).contiguous()

        def bn(p, use_bn):
            if use_bn:
                s, t = L.fold_bn(sd, p + ".batch_norm", BN_EPS)
                put(p + ".s", s), put(p + ".t", t)
            else:
                put(p + ".t", sd[p + ".bias"])

        def unary(p, use_bn):
            w[p + ".wt"] = L.pack_linear(sd[p + ".mlp.weight"].t())
            bn(p + ".batch_norm", use_bn)

        def kpconv(p, deform):
            kw = sd[p + ".weights"]  # [K, Cin, Cout]
            w[p + ".wt"] = L.pack_linear(kw.reshape(kw.shape[0] * kw.shape[1], kw.shape[2]))
            if not deform:
                put(p + ".kp", sd[p + ".kernel_points"])
                return
            # KPConv.kernel_points IS offset_conv.kernel_points (kpconv.py:977-978): one Parameter under two keys,
            # and load_state_dict loads the child last, so the offset_conv value is the one the module uses
            put(p + ".kp", sd[p + ".offset_conv.kernel_points"])
            ow = sd[p + ".offset_conv.weights"]  # [K, Cin, 3K]
            w[p + ".off_wt"] = L.pack_linear(ow.reshape(ow.shape[0] * ow.shape[1], ow.shape[2]))
            put(p + ".off_t", sd[p + ".offset_bias"])

        for bi, b in enumerate(self.enc):
            p = "encoder_blocks.%d" % bi
            kpconv(p + ".KPConv", b["deform"])
            if "simple" in b["kind"]:
                bn(p + ".batch_norm", self.use_bn)
            else:
                if b["in_dim"] != b["out_dim"] // 4:
                    unary(p + ".unary1", self.use_bn)
                bn(p + ".batch_norm_conv", self.use_bn)
                unary(p + ".unary2", self.use_bn)
                if b["in_dim"] != b["out_dim"]:
                    unary(p + ".unary_shortcut", self.use_bn)
        for bi, b in enumerate(self.dec):
            if b["kind"] == "unary":
                unary("decoder_blocks.%d" % bi, self.use_bn)
        # kpconv.py:228-249: reduce_fc -> head_mlp with BN, head_softmax without activation
        self.reduce_fc = bool(cfg.get("reduce_fc", False))
        unary("head_mlp", self.reduce_fc and self.use_bn)
        unary("head_softmax", False)
        self.num_classes = sd["head_softmax.mlp.weight"].shape[0]

    def _lin(self, p, srcs, n, act, residual=None):
        wt = self.w[p + ".wt"]
        out = torch.empty((n, wt.shape[1]), dtype=torch.float32, device=self.device)
        return L.linear(srcs, wt, out, self.w.get(p + ".batch_norm.s"), self.w[p + ".batch_norm.t"],
                        residual=residual, act=act, slope=self.slope)

    def _kpconv(self, p, q_pts, s_pts, nidx, x, extent, bn_name, deform=False, probe=None):
        kp = self.w[p + ".kp"]
        K, cin = kp.shape[0], x.shape[1]
        nq = q_pts.shape[0]
        is64 = L.is64(nidx)
        events = []

        def mark():
            if probe is not None and deform:
                events.append(torch.cuda.Event(enable_timing=True))
                events[-1].record()
        mark()
        a = torch.empty((nq, K * cin), dtype=torch.float32, device=self.device)
        L.check(L.lib().o3dml_kpconv_gather(
            L.ptr(q_pts), nq, L.ptr(s_pts), s_pts.shape[0], L.ptr(nidx), is64, nidx.shape[1], L.ptr(x), cin,
            L.ptr(kp), K, float(extent), L.ptr(a), L.stream()))
        if deform:
            # offset conv (a rigid KPConv with 3K outputs, no BN / activation) + offset_bias, in 48-float rows
            # (16-byte aligned); then the deformable gather overwrites `a` in stream order
            mark()
            off = torch.empty((nq, 48), dtype=torch.float32, device=self.device)
            L.linear([L.make_src(a)], self.w[p + ".off_wt"], off, None, self.w[p + ".off_t"])
            mark()
            L.check(L.lib().o3dml_kpconv_gather_deformable(
                L.ptr(q_pts), nq, L.ptr(s_pts), s_pts.shape[0], L.ptr(nidx), is64, nidx.shape[1], L.ptr(x), cin,
                L.ptr(kp), K, float(extent), L.ptr(off), off.stride(0), L.ptr(a), L.stream()))
            mark()
        wt = self.w[p + ".wt"]
        out = torch.empty((nq, wt.shape[1]), dtype=torch.float32, device=self.device)
        L.linear([L.make_src(a)], wt, out, self.w.get(bn_name + ".s"), self.w[bn_name + ".t"],
                 act="leaky", slope=self.slope)
        mark()
        if probe is not None and deform:
            probe.append(dict(name=p, events=events, offsets=off[:, :3 * K], kernel_points=kp, extent=float(extent),
                              q_pts=q_pts, s_pts=s_pts, neighbors=nidx))
        return out

    def forward(self, batch, taps=None, probe=None):
        """`taps` (dict) receives every block's output.  `probe` (list) receives, for every deformable KPConv, its
        name, its inputs, its offsets and CUDA events around its four steps (offset gather, offset GEMM,
        deformable gather, GEMM): what bench_kpconv_deform.py reports."""
        dev = self.device

        def mv(t):
            return t.to(dev, non_blocking=True).contiguous()
        if isinstance(batch, dict):
            g = batch.__getitem__
        else:
            g = lambda k: getattr(batch, k)  # noqa: E731
        pts = [mv(t).float() for t in g("points")]
        nbr = [mv(t) for t in g("neighbors")]
        pools = [mv(t) for t in g("pools")]
        ups = [mv(t) for t in g("upsamples")]
        x = mv(g("features")).float()
        skip_x = []
        for bi, b in enumerate(self.enc):
            p = "encoder_blocks.%d" % bi
            if bi in self.enc_skips:
                skip_x.append(x)
            lay = b["layer"]
            strided = "strided" in b["kind"]
            q = pts[lay + 1] if strided else pts[lay]
            s = pts[lay]
            nidx = pools[lay] if strided else nbr[lay]
            if "simple" in b["kind"]:
                x = self._kpconv(p + ".KPConv", q, s, nidx, x, b["extent"], p + ".batch_norm", b["deform"], probe)
            else:
                feats = x
                y = feats
                if b["in_dim"] != b["out_dim"] // 4:
                    y = self._lin(p + ".unary1", [L.make_src(y)], y.shape[0], "leaky")
                y = self._kpconv(p + ".KPConv", q, s, nidx, y, b["extent"], p + ".batch_norm_conv", b["deform"],
                                 probe)
                sc = feats
                if strided:
                    sc = torch.empty((q.shape[0], feats.shape[1]), dtype=torch.float32, device=dev)
                    L.check(L.lib().o3dml_gather_max(
                        L.ptr(feats), feats.shape[0], feats.shape[1], feats.stride(0), L.ptr(nidx), L.is64(nidx),
                        q.shape[0], nidx.shape[1], 0, 0, 1, L.ptr(sc), sc.stride(0), L.stream()))
                if b["in_dim"] != b["out_dim"]:
                    sc = self._lin(p + ".unary_shortcut", [L.make_src(sc)], sc.shape[0], None)
                x = self._lin(p + ".unary2", [L.make_src(y)], y.shape[0], "leaky", residual=sc)
            if taps is not None:
                taps[p] = x
        pending = None  # (index tensor) of a nearest_upsample waiting to be fused
        for bi, b in enumerate(self.dec):
            p = "decoder_blocks.%d" % bi
            skip = skip_x.pop() if bi in self.dec_concats else None
            if "upsample" in b["kind"]:
                if pending is not None:
                    raise RuntimeError("KPFCNNB200: two upsample blocks in a row")
                pending = ups[b["layer"] - 1]
            elif b["kind"] == "unary":
                n = pending.shape[0] if pending is not None else x.shape[0]
                src0 = (L.make_src(x, index=pending, index_ld=pending.shape[1])
                        if pending is not None else L.make_src(x))
                srcs = [src0] + ([L.make_src(skip)] if skip is not None else [])
                x = self._lin(p, srcs, n, "leaky")
                pending = None
            else:
                raise RuntimeError("KPFCNNB200: decoder block '%s' not supported" % b["kind"])
            if taps is not None and pending is None:
                taps[p] = x
        if pending is not None:
            raise RuntimeError("KPFCNNB200: dangling upsample block")
        x = self._lin("head_mlp", [L.make_src(x)], x.shape[0], "leaky")
        return self._lin("head_softmax", [L.make_src(x)], x.shape[0], None if self.reduce_fc else "leaky")

    __call__ = forward


def patch_reference_model(model):
    """Drop-in: make an (unmodified) reference ``KPFCNN`` instance run its forward on the fused CUDA path (keeps
    preprocess / transform / losses, ``inference_*`` and ``update_probs``).  Built from ``model.state_dict()`` and
    ``model.cfg``, so ``reduce_fc``, ``l_relu``, ``use_batch_norm`` and the architecture are the ones the model was
    built with; BN must be in eval mode.  The fused weights are a snapshot taken here: patch again after loading new
    ones.  The batch is the reference ``KPConvBatch`` (its geometry still comes from the reference batcher), on the
    CPU or the device; the result is ``[sum N_i, num_classes]`` float32 on the device.  A config the fused path does
    not build (``modulated`` deformable KPConv, another ``KP_influence`` or ``aggregation_mode``) raises here and
    leaves ``model.forward`` as it was."""
    fused = KPFCNNB200(model.state_dict(), dict(model.cfg))

    def forward(batch):
        if model.training:
            raise RuntimeError("open3d_ml_b200: the fused KPFCNN path is inference-only")
        return fused.forward(batch)
    model.forward = forward
    return model


def layer_radii(cfg):
    """[(conv, pool, upsample)] search radius of every layer, as KPConvBatch.segmentation_inputs picks them
    (ml3d/torch/dataloaders/concat_batcher.py:209-262): r = first_subsampling_dl * conv_radius doubling per layer;
    the conv neighbours use r * deform_radius / conv_radius when a block of the layer before its closing block is
    deformable, the pool neighbours when the closing block is, and the upsample neighbours twice the pool radius.
    The KPConv extents keep the normal r (kpconv.py:1376)."""
    r = cfg["first_subsampling_dl"] * cfg["conv_radius"]
    out, blocks = [], []
    for blk in cfg["architecture"]:
        if not any(t in blk for t in ("pool", "strided", "global", "upsample")):
            blocks.append(blk)
            continue
        deform_r = r * cfg.get("deform_radius", 6.0) / cfg["conv_radius"]     # KPFCNN's default (kpconv.py:61)
        conv = deform_r if any("deformable" in b for b in blocks) else r
        pool = deform_r if "deformable" in blk else r
        out.append((conv, pool, 2 * pool))
        r *= 2
        blocks = []
        if "global" in blk or "upsample" in blk:
            break
    return out


def build_batch(clouds, cfg, device="cuda", neighborhood_limits=None, timings=None):
    """KPConvBatch.segmentation_inputs (ml3d/torch/dataloaders/concat_batcher.py:186-305) on the device for a
    list of (points [n,3], features [n,F]) numpy clouds: the clouds are stacked once, then per level
      conv neighbours   batch_neighbors(P, P, r)            (kpconv.py:2002-2034)
      sub-sampled cloud batch_grid_subsampling(P, dl = 2 r / conv_radius), barycentre per voxel (:2037-2164)
      pool / upsample   batch_neighbors(Q, P, r), batch_neighbors(P, Q, 2 r)
    all with the CUDA fixed-radius search / voxelize / voxel_reduce kernels (13 searches + 4 subsamplings for
    the 5-level S3DIS config) at the radii of `layer_radii`, padded with the shadow id and cropped by `neighborhood_limits` like
    big_neighborhood_filter (:175-186).  Returns a dict of CUDA tensors (indices int64 as the reference)."""
    import numpy as np
    from . import ops

    def neighbors(queries, supports, qs, ss, radius, limit=None):
        r = ops.fixed_radius_search(supports, queries, radius, ss, qs, return_distances=False)
        rs = r.neighbors_row_splits
        width = int((rs[1:] - rs[:-1]).max()) if rs.numel() > 1 else 0
        if limit is not None:
            width = min(width, int(limit))
        return ops.ragged_to_dense(r.neighbors_index, rs, width,
                                   torch.tensor([supports.shape[0]], dtype=torch.int32)).to(torch.int64)

    lim = list(neighborhood_limits) if neighborhood_limits else None
    radii = layer_radii(cfg)
    r = cfg["first_subsampling_dl"] * cfg["conv_radius"]
    out = dict(features=torch.from_numpy(np.concatenate([c[1] for c in clouds])).to(device),
               points=[], neighbors=[], pools=[], upsamples=[], lengths=[])
    P = torch.from_numpy(np.concatenate([c[0] for c in clouds]).astype(np.float32)).to(device)
    rs = torch.tensor(np.concatenate([[0], np.cumsum([len(c[0]) for c in clouds])]), dtype=torch.int64,
                      device=device)
    for lvl in range(cfg["num_layers"]):
        out["points"].append(P)
        out["lengths"].append((rs[1:] - rs[:-1]).to(torch.int32))
        conv_r, pool_r, up_r = radii[lvl]
        out["neighbors"].append(neighbors(P, P, rs, rs, conv_r, lim[lvl] if lim else None))
        if lvl < cfg["num_layers"] - 1:
            dl = 2 * r / cfg["conv_radius"]
            Q, qs, _, _ = ops.subsample_batch_cuda(P, rs, sampleDl=dl)
            out["pools"].append(neighbors(Q, P, qs, rs, pool_r, lim[lvl] if lim else None))
            out["upsamples"].append(neighbors(P, Q, rs, qs, up_r, lim[lvl + 1] if lim else None))
            P, rs, r = Q, qs, r * 2
        else:
            out["pools"].append(torch.zeros((0, 1), dtype=torch.int64, device=device))
            out["upsamples"].append(torch.zeros((0, 1), dtype=torch.int64, device=device))
    return out
