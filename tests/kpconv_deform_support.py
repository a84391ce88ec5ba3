"""Torch restatement of the deformable KPConv and of the KPFCNN forward that uses it (test support, CPU or GPU).

It extends oracle/models_torch.py's rigid KPFCNN port, whose existing functions keep their results:
  KPConv.forward, deformable, modulated = False   ml3d/torch/models/kpconv.py:1011-1159
  KPFCNN head with reduce_fc                       kpconv.py:219-241
The deformable conv and the offset conv both use KPConv.offset_conv.kernel_points: KPConv.kernel_points is the
same Parameter (kpconv.py:977-978), and load_state_dict loads the child's key last.
tests/ref_kpconv_deform_case.py pins kpfcnn_forward here against the unmodified reference class.
"""
import torch

from oracle import models_torch as MT


def deformed_kernel_points(q_pts, s_pts, nidx, x, kpts, off_weights, off_bias, extent):
    """The offset conv (a rigid KPConv with 3K outputs) + offset_bias, scaled by the extent and added to the
    kernel points, each step rounded on its own: -> [Nq, K, 3] in the dtype of the inputs."""
    off = MT.kp_conv(q_pts, s_pts, nidx, x, kpts, off_weights, extent) + off_bias
    return off.view(-1, kpts.shape[0], 3) * extent + kpts


def deform_influence(q_pts, s_pts, nidx, dkp, extent):
    """-> (weights [Nq, K, H], kept [Nq, H]): the linear influence of the per-query kernel points dkp [Nq, K, 3]
    and the re-selection of kpconv.py:1071-1103 (kept: d2 < extent^2 for some kernel point)."""
    s_pts = torch.cat([s_pts, torch.full_like(s_pts[:1], 1e6)])
    nb = s_pts[nidx] - q_pts.unsqueeze(1)                       # [Nq, H, 3]
    diff = nb.unsqueeze(2) - dkp.unsqueeze(1)                   # [Nq, H, K, 3]
    d2 = (diff * diff).sum(-1)
    kept = (d2 < extent ** 2).any(2)
    w = torch.clamp(1 - torch.sqrt(d2) / extent, min=0.0).transpose(1, 2)
    return w, kept


def deform_gather(q_pts, s_pts, nidx, x, dkp, extent):
    """The [Nq, K, Cin] operand of a deformable KPConv: dropped neighbours read the shadow (zero) feature, so a
    non-finite feature of a dropped neighbour does not reach the sum, while one of a kept neighbour does."""
    w, kept = deform_influence(q_pts, s_pts, nidx, dkp, extent)
    idx = torch.where(kept, nidx, torch.full_like(nidx, s_pts.shape[0]))
    x = torch.cat([x, torch.zeros_like(x[:1])])
    return w @ x[idx]


def kp_conv_deform(q_pts, s_pts, nidx, x, sd, p, extent, stats=None):
    """Deformable KPConv.forward (kpconv.py:1011-1159) from the state_dict keys under `p` (…KPConv)."""
    kpts = sd[p + ".offset_conv.kernel_points"]
    dkp = deformed_kernel_points(q_pts, s_pts, nidx, x, kpts, sd[p + ".offset_conv.weights"],
                                 sd[p + ".offset_bias"], extent)
    wf = deform_gather(q_pts, s_pts, nidx, x, dkp, extent)
    if stats is not None:
        _, kept = deform_influence(q_pts, s_pts, nidx, dkp, extent)
        valid = (nidx >= 0) & (nidx < s_pts.shape[0])
        stats[p] = dict(kept=int(kept.sum()), dropped=int((valid & ~kept).sum()),
                        median_offset=float((dkp - kpts).norm(dim=-1).median()) / extent)
    return torch.einsum("nkc,kcd->nd", wf, sd[p + ".weights"])


def kpfcnn_forward(sd, batch, cfg, taps=None, stats=None):
    """KPFCNN.forward (kpconv.py:270-291) with rigid and deformable blocks and either head."""
    plan = MT.kpfcnn_plan(cfg)
    use_bn, slope = cfg.get("use_batch_norm", True), cfg.get("l_relu", 0.1)
    x = batch["features"]
    skip_x = []

    def conv(p, q, s, nidx, y, b):
        if "deform" in b["kind"]:
            return kp_conv_deform(q, s, nidx, y, sd, p + ".KPConv", b["extent"], stats)
        return MT.kp_conv(q, s, nidx, y, sd[p + ".KPConv.kernel_points"], sd[p + ".KPConv.weights"], b["extent"])

    for bi, b in enumerate(plan["encoder"]):
        p = "encoder_blocks.%d" % bi
        if bi in plan["encoder_skips"]:
            skip_x.append(x)
        lay = b["layer"]
        strided = "strided" in b["kind"]
        q = batch["points"][lay + 1] if strided else batch["points"][lay]
        s = batch["points"][lay]
        nidx = batch["pools"][lay] if strided else batch["neighbors"][lay]
        if "simple" in b["kind"]:
            x = MT.lrelu(MT.kp_bn(conv(p, q, s, nidx, x, b), sd, p + ".batch_norm", use_bn), slope)
        elif "resnetb" in b["kind"]:
            feats = x
            y = feats
            if b["in_dim"] != b["out_dim"] // 4:
                y = MT.kp_unary(y, sd, p + ".unary1", use_bn, True, slope)
            y = MT.lrelu(MT.kp_bn(conv(p, q, s, nidx, y, b), sd, p + ".batch_norm_conv", use_bn), slope)
            y = MT.kp_unary(y, sd, p + ".unary2", use_bn, False, slope)
            sc = MT.kp_max_pool(feats, nidx) if strided else feats
            if b["in_dim"] != b["out_dim"]:
                sc = MT.kp_unary(sc, sd, p + ".unary_shortcut", use_bn, False, slope)
            x = MT.lrelu(y + sc, slope)
        else:
            raise NotImplementedError(b["kind"])
        if taps is not None:
            taps[p] = x
    for bi, b in enumerate(plan["decoder"]):
        p = "decoder_blocks.%d" % bi
        if bi in plan["decoder_concats"]:
            x = torch.cat([x, skip_x.pop()], 1)
        if "upsample" in b["kind"]:
            x = MT.kp_closest_pool(x, batch["upsamples"][b["layer"] - 1])
        elif b["kind"] == "unary":
            x = MT.kp_unary(x, sd, p, use_bn, True, slope)
        else:
            raise NotImplementedError(b["kind"])
        if taps is not None:
            taps[p] = x
    if cfg.get("reduce_fc", False):
        # kpconv.py:229-241: head_mlp with BN (always) and LeakyReLU, head_softmax with a bias and no activation
        x = MT.kp_unary(x, sd, "head_mlp", True, True, slope)
        return MT.kp_unary(x, sd, "head_softmax", False, False, slope)
    # kpconv.py:242-249: both head UnaryBlocks without BN and with LeakyReLU
    x = MT.kp_unary(x, sd, "head_mlp", False, True, slope)
    return MT.kp_unary(x, sd, "head_softmax", False, True, slope)


def paris_clouds(seed, batch_limit=20000, in_radius=4.0, dl=0.08, n=200000):
    """Paris-Lille3D-shaped input: 4 m spheres cropped from synthetic LiDAR frames around points within 15 m of the
    sensor, grid-subsampled at 0.08 m (features: the constant 1 of in_features_dim = 1) and stacked while the total
    stays within batch_limit points.  -> list of (points [n,3], features [n,1]) float32 numpy clouds."""
    import numpy as np
    from open3d_ml_b200 import synth
    rng = np.random.default_rng(seed)
    clouds, total = [], 0
    for s in range(seed, seed + 64):
        pc = synth.semantickitti_cloud(n, s)
        near = pc[np.linalg.norm(pc[:, :2], axis=1) < 15.0]
        c = near[rng.integers(len(near))]
        crop = pc[np.linalg.norm(pc - c, axis=1) < in_radius] - c
        pts = synth.grid_subsample(crop, dl).astype(np.float32)
        if total + len(pts) > batch_limit:
            break
        clouds.append((pts, np.ones((len(pts), 1), np.float32)))
        total += len(pts)
    return clouds
