"""oracle/models_torch.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Plain-PyTorch (CPU, float32) restatement of the three reference forwards on the
hot path, driven by the reference's own ``state_dict`` keys, in point-major
(channels-last) layout.  It is the one port of the reference in the repository:
it exists because the reference tree does not travel to the GPU machines.
tests/test_oracle_models.py, test_oracle_kpconv_deform.py and
test_oracle_pointpillars_configs.py pin it against the UNMODIFIED reference
classes (imported through oracle/refshim.py) where the reference is installed,
and against the committed golden fixtures everywhere.  On a GPU it is the parity
checker for full-size inputs, the kernel tests' float64 reference and the
"port" CPU baseline.

Reference lines followed:
  RandLANet.forward            ml3d/torch/models/randlanet.py:241-298
  SharedMLP                    randlanet.py:471-518
  LocalSpatialEncoding         randlanet.py:521-605
  AttentivePooling             randlanet.py:608-639
  LocalFeatureAggregation      randlanet.py:642-692
  random_sample / nearest_interpolation   randlanet.py:300-350
  PointPillars.forward         ml3d/torch/models/point_pillars.py:102-134
  PointPillarsVoxelization     point_pillars.py:328-382
  PillarFeatureNet / PFNLayer  point_pillars.py:400-555 (one or more layers)
  PointPillarsScatter          point_pillars.py:577-616
  SECOND / SECONDFPN / head    point_pillars.py:619-841
  KPFCNN.forward               ml3d/torch/models/kpconv.py:270-291
  KPFCNN heads (reduce_fc or not)   kpconv.py:229-251
  KPConv.forward (rigid and deformable, modulated = False)   kpconv.py:1005-1159
  Unary/Resnet/Simple blocks   kpconv.py:1213-1464, max_pool/closest_pool :821-858

Only tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / ``--impl reference``
legs and the side benches (bench_kpconv_deform.py) may import this module.
"""
import itertools
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import ops as O


def lrelu(x, slope):
    return torch.where(x >= 0, x, x * slope)


def bn_eval(x, sd, prefix, eps):
    """Eval-mode batch norm on the LAST axis of x."""
    s = sd[prefix + ".weight"] / torch.sqrt(sd[prefix + ".running_var"] + eps)
    return (x - sd[prefix + ".running_mean"]) * s + sd[prefix + ".bias"]


# =============================================================================
# RandLA-Net
# =============================================================================
RANDLA_BN_EPS = 1e-6  # randlanet.py:77,499


def rl_shared_mlp(x, sd, p, slope=None, bn=True, transpose=False):
    """1x1 (transposed) conv with bias + BN + LeakyReLU on [..., Cin] (randlanet.py:471-518)."""
    w = sd[p + ".conv.weight"][:, :, 0, 0]
    w = w if transpose else w.t()  # -> [Cin, Cout]
    y = x @ w + sd[p + ".conv.bias"]
    if bn:
        y = bn_eval(y, sd, p + ".batch_norm", RANDLA_BN_EPS)
    return y if slope is None else lrelu(y, slope)


def rl_gather(feat, idx):
    """feat [B,N,C], idx [B,M,K] -> [B,M,K,C] (randlanet.py:533-553)."""
    B, M, K = idx.shape
    flat = idx.reshape(B, M * K, 1).expand(-1, -1, feat.shape[-1])
    return torch.gather(feat, 1, flat).reshape(B, M, K, feat.shape[-1])


def rl_attentive_pool(x, sd, p):
    """x [B,N,K,d] -> [B,N,d_out] (randlanet.py:608-639)."""
    s = x @ sd[p + ".score_fn.0.weight"].t() + sd[p + ".score_fn.0.bias"]
    s = torch.softmax(s, dim=2)  # over K
    agg = (s * x).sum(dim=2)
    return rl_shared_mlp(agg, sd, p + ".mlp", 0.2)


def rl_relative_features(coords, nidx):
    """10-channel encoding [dist, centre-neighbour, centre, neighbour] (randlanet.py:575-592)."""
    nb = rl_gather(coords, nidx)  # [B,N,K,3]
    ctr = coords.unsqueeze(2).expand_as(nb)
    rel = ctr - nb
    dist = torch.sqrt((rel * rel).sum(-1, keepdim=True))
    return torch.cat([dist, rel, ctr, nb], dim=-1)


def rl_lfa(coords, feat, nidx, sd, p, taps=None):
    """LocalFeatureAggregation: feat [B,N,d_in] -> [B,N,2*d_out] (randlanet.py:667-692)."""
    x = rl_shared_mlp(feat, sd, p + ".mlp1", 0.2)
    r1 = rl_shared_mlp(rl_relative_features(coords, nidx), sd, p + ".lse1.mlp", 0.2)
    x = rl_attentive_pool(torch.cat([rl_gather(x, nidx), r1], -1), sd, p + ".pool1")
    if taps is not None:
        taps[p + ".pool1"] = x
    r2 = rl_shared_mlp(r1, sd, p + ".lse2.mlp", 0.2)
    x = rl_attentive_pool(torch.cat([rl_gather(x, nidx), r2], -1), sd, p + ".pool2")
    y = rl_shared_mlp(x, sd, p + ".mlp2") + rl_shared_mlp(feat, sd, p + ".shortcut")
    return lrelu(y, 0.01)


def randlanet_forward(sd, inputs, num_layers=4, taps=None):
    """inputs: dict(features [B,N,Cin], coords[i] [B,N_i,3], neighbor_indices[i] [B,N_i,K],
    sub_idx[i] [B,N_i/4,K], interp_idx[i] [B,N_i,1]) -> logits [B,N,classes]."""
    feat = inputs["features"] @ sd["fc0.weight"].t() + sd["fc0.bias"]
    feat = lrelu(bn_eval(feat, sd, "bn0", RANDLA_BN_EPS), 0.2)
    skips = []
    for i in range(num_layers):
        enc = rl_lfa(inputs["coords"][i], feat, inputs["neighbor_indices"][i], sd,
                     "encoder.%d" % i, taps)
        if taps is not None:
            taps["encoder.%d" % i] = enc
        sub = rl_gather(enc, inputs["sub_idx"][i]).max(dim=2)[0]  # random_sample :300-327
        if i == 0:
            skips.append(enc)
        skips.append(sub)
        feat = sub
    feat = rl_shared_mlp(feat, sd, "mlp", 0.2)
    for i in range(num_layers):
        up = rl_gather(feat, inputs["interp_idx"][-i - 1])[:, :, 0, :]  # nearest_interpolation
        feat = rl_shared_mlp(torch.cat([skips[-i - 2], up], -1), sd, "decoder.%d" % i, 0.2,
                             transpose=True)
        if taps is not None:
            taps["decoder.%d" % i] = feat
    feat = rl_shared_mlp(feat, sd, "fc1.0", 0.2)
    feat = rl_shared_mlp(feat, sd, "fc1.1", 0.2)
    return rl_shared_mlp(feat, sd, "fc1.3", None, bn=False)  # fc1.2 = Dropout (eval: identity)


def randlanet_build_inputs(pc, num_layers=4, k=16, ratios=(4, 4, 4, 4), knn=None):
    """KNN pyramid of RandLANet.transform (randlanet.py:218-229) for one cloud [N,3].
    Returns numpy arrays without the batch axis."""
    knn = knn or (lambda s, q, kk: O.np_knn(s, q, kk)[0])
    out = dict(coords=[], neighbor_indices=[], sub_idx=[], interp_idx=[])
    for i in range(num_layers):
        nb = knn(pc, pc, k)
        n_sub = pc.shape[0] // ratios[i]
        sub = pc[:n_sub]
        out["coords"].append(pc)
        out["neighbor_indices"].append(nb.astype(np.int64))
        out["sub_idx"].append(nb[:n_sub].astype(np.int64))
        out["interp_idx"].append(knn(sub, pc, 1).astype(np.int64))
        pc = sub
    return out


# =============================================================================
# PointPillars
# =============================================================================
PP_BN_EPS = 1e-3  # point_pillars.py:409,648,724


def pp_grid(point_cloud_range, voxel_size):
    """float32 grid extent as computed at point_pillars.py:352-353."""
    r = torch.tensor(point_cloud_range, dtype=torch.float32)
    v = torch.tensor(voxel_size, dtype=torch.float32)
    return ((r[3:] - r[:3]) / v).to(torch.int32)


def pp_voxelize(points, cfg, voxelize=None):
    """One frame [N,C>=3] -> (pillars [M,P,C], coords [M,3] (z,y,x) int32, counts [M])
    (point_pillars.py:328-382)."""
    voxelize = voxelize or O.c_voxelize
    r = cfg["point_cloud_range"]
    ans = voxelize(points[:, :3].contiguous().numpy(), np.array([0, points.shape[0]], np.int64),
                   np.float32(cfg["voxel_size"]), np.float32(r[:3]), np.float32(r[3:]),
                   cfg["max_num_points"], cfg["max_voxels"])
    P = cfg["max_num_points"]
    dense = O.np_ragged_to_dense(ans["voxel_point_indices"], ans["voxel_point_row_splits"], P,
                                 np.int64(-1)) + 1
    feats = torch.cat([torch.zeros_like(points[:1]), points])
    pillars = feats[torch.from_numpy(dense)]
    coords = torch.from_numpy(ans["voxel_coords"][:, [2, 1, 0]].copy())
    rs = torch.from_numpy(ans["voxel_point_row_splits"])
    counts = rs[1:] - rs[:-1]
    g = pp_grid(r, cfg["voxel_size"])
    ok = (coords[:, 1] < g[1]) & (coords[:, 2] < g[0])
    return pillars[ok], coords[ok], counts[ok]


def pp_decorate(pillars, counts, cx, cy, vx, vy, x_off, y_off):
    """PillarFeatureNet's decoration (point_pillars.py:512-555): pillars [M,P,C] with counts [M] points and cell
    x / y [M] -> [M,P,C+5] = [point, point - pillar mean (f_cluster), x / y - cell centre (f_center)], the padded
    slots zeroed."""
    cnt = counts.to(pillars.dtype).view(-1, 1, 1)
    mean = pillars[:, :, :3].sum(1, keepdim=True) / cnt
    f_cluster = pillars[:, :, :3] - mean
    f_center = torch.stack([
        pillars[:, :, 0] - (cx.to(pillars.dtype).unsqueeze(1) * vx + x_off),
        pillars[:, :, 1] - (cy.to(pillars.dtype).unsqueeze(1) * vy + y_off)], -1)
    f = torch.cat([pillars, f_cluster, f_center], -1)
    slot = torch.arange(pillars.shape[1], device=pillars.device).view(1, -1)
    return f * (slot < counts.view(-1, 1)).unsqueeze(-1).to(f.dtype)


def pp_pfn(pillars, counts, coords4, sd, cfg):
    """PillarFeatureNet with its PFNLayers: -> [M,64] (point_pillars.py:400-555).  Only the decoration is masked:
    every slot, padded ones included, takes part in every layer's max (SURVEY.md A1), and a layer that is not the
    last passes cat(y[p], max over slots of y) on."""
    vx, vy = cfg["voxel_size"][0], cfg["voxel_size"][1]
    f = pp_decorate(pillars, counts, coords4[:, 3], coords4[:, 2], vx, vy,
                    vx / 2 + cfg["point_cloud_range"][0], vy / 2 + cfg["point_cloud_range"][1])
    for i in itertools.count():
        p = "voxel_encoder.pfn_layers.%d" % i
        y = torch.relu(bn_eval(f @ sd[p + ".linear.weight"].t(), sd, p + ".norm", PP_BN_EPS))
        m = y.max(dim=1, keepdim=True)[0]
        if "voxel_encoder.pfn_layers.%d.linear.weight" % (i + 1) not in sd:
            return m.squeeze(1)
        f = torch.cat([y, m.expand_as(y)], 2)


def pp_scatter(vfeat, coords4, batch, ny, nx):
    """-> canvas [B,C,ny,nx] (point_pillars.py:577-616)."""
    C = vfeat.shape[1]
    canvas = torch.zeros(batch, C, ny * nx, dtype=vfeat.dtype)
    lin = (coords4[:, 2].long() * nx + coords4[:, 3].long())
    canvas[coords4[:, 0].long(), :, lin] = vfeat
    return canvas.view(batch, C, ny, nx)


def pp_conv_bn_relu(x, sd, conv, bn, stride=1, padding=1):
    y = F.conv2d(x, sd[conv + ".weight"], None, stride, padding)
    y = bn_eval(y.permute(0, 2, 3, 1), sd, bn, PP_BN_EPS).permute(0, 3, 1, 2)
    return torch.relu(y)


def pp_backbone_neck_head(x, sd, cfg):
    """SECOND + SECONDFPN + Anchor3DHead (point_pillars.py:669-682,739-755,827-841)."""
    outs = []
    for i, (n, s) in enumerate(zip(cfg["layer_nums"], cfg["layer_strides"])):
        p = "backbone.blocks.%d" % i
        x = pp_conv_bn_relu(x, sd, p + ".0", p + ".1", stride=s)
        for j in range(n):
            x = pp_conv_bn_relu(x, sd, "%s.%d" % (p, 3 + 3 * j), "%s.%d" % (p, 4 + 3 * j))
        outs.append(x)
    ups = []
    for i, s in enumerate(cfg["upsample_strides"]):
        p = "neck.deblocks.%d" % i
        y = F.conv_transpose2d(outs[i], sd[p + ".0.weight"], None, stride=s)
        y = bn_eval(y.permute(0, 2, 3, 1), sd, p + ".1", PP_BN_EPS).permute(0, 3, 1, 2)
        ups.append(torch.relu(y))
    f = torch.cat(ups, 1)
    return tuple(F.conv2d(f, sd["bbox_head.%s.weight" % h], sd["bbox_head.%s.bias" % h])
                 for h in ("conv_cls", "conv_reg", "conv_dir_cls"))


def pointpillars_forward(sd, frames, cfg, voxelize=None, taps=None):
    """frames: list of [N_i,4] float32 tensors -> (cls, reg, dir) NCHW."""
    pil, co, cn = [], [], []
    for b, pts in enumerate(frames):
        p, c, n = pp_voxelize(pts, cfg, voxelize)
        pil.append(p)
        co.append(F.pad(c, (1, 0), value=b))
        cn.append(n)
    pil, co, cn = torch.cat(pil), torch.cat(co), torch.cat(cn)
    vf = pp_pfn(pil, cn, co, sd, cfg)
    ny, nx = cfg["output_shape"]
    canvas = pp_scatter(vf, co, len(frames), ny, nx)
    if taps is not None:
        taps.update(pillars=pil, coords=co, counts=cn, pfn=vf, canvas=canvas)
    return pp_backbone_neck_head(canvas, sd, cfg)


# =============================================================================
# KPConv / KPFCNN (linear influence, sum aggregation: SURVEY.md A11; rigid and deformable, not modulated)
# =============================================================================
KP_BN_EPS = 1e-5  # nn.BatchNorm1d default (kpconv.py:1231)


def kp_d2(q_pts, s_pts, nidx, kpts):
    """[Nq,H,K] squared distances of the neighbours nidx [Nq,H], relative to their query, to the kernel points kpts:
    [K,3] (rigid) or [Nq,K,3] (deformed, per query).  Every id outside [0, ns) reads the shadow point at 1e6."""
    ns = s_pts.shape[0]
    s_pts = torch.cat([s_pts, torch.full_like(s_pts[:1], 1e6)])
    nb = s_pts[torch.where((nidx >= 0) & (nidx < ns), nidx, ns)] - q_pts.unsqueeze(1)  # [Nq,H,3]
    diff = nb.unsqueeze(2) - kpts.unsqueeze(-3)  # [Nq,H,K,3]
    return (diff * diff).sum(-1)


def kp_kept(q_pts, s_pts, nidx, kpts, extent):
    """The deformable conv's re-selection (kpconv.py:1071-1103): [Nq,H], true where d2 < extent^2 for some kernel
    point."""
    return (kp_d2(q_pts, s_pts, nidx, kpts) < extent ** 2).any(2)


def kp_gather(q_pts, s_pts, nidx, x, kpts, extent, keep=None):
    """The [Nq,K,Cin] operand of KPConv.forward (kpconv.py:1044-1159): sum over the neighbours n of
    max(0, 1 - |s[n] - q - kp| / extent) * x[n].  Ids outside [0, ns) and the neighbours that keep [Nq,H] drops read
    the shadow row, whose feature is zero: a non-finite feature of a dropped neighbour does not reach the sum."""
    ns = s_pts.shape[0]
    w = torch.clamp(1 - torch.sqrt(kp_d2(q_pts, s_pts, nidx, kpts)) / extent, min=0.0).transpose(1, 2)  # [Nq,K,H]
    ok = (nidx >= 0) & (nidx < ns)
    if keep is not None:
        ok = ok & keep
    x = torch.cat([x, torch.zeros_like(x[:1])])
    return w @ x[torch.where(ok, nidx, ns)]


def kp_conv(q_pts, s_pts, nidx, x, kpts, weights, extent, keep=None):
    """KPConv.forward: the gathered operand contracted with weights [K,Cin,Cout]."""
    return torch.einsum("nkc,kcd->nd", kp_gather(q_pts, s_pts, nidx, x, kpts, extent, keep), weights)


def kp_conv_deform(q_pts, s_pts, nidx, x, sd, p, extent, stats=None):
    """Deformable KPConv.forward (kpconv.py:1011-1159) from the state_dict keys under p (...KPConv).  The offset conv
    (a rigid KPConv with 3K outputs) + offset_bias, scaled by the extent and added to the kernel points, each step
    rounded on its own, moves the kernel points per query; the conv then re-selects and gathers at the moved points.
    Both convs read offset_conv.kernel_points: KPConv.kernel_points is the same Parameter (kpconv.py:977-978), and
    load_state_dict loads the child's key last.  stats[p] gets the kept / dropped valid neighbours and the median
    offset in extents."""
    kpts = sd[p + ".offset_conv.kernel_points"]
    off = kp_conv(q_pts, s_pts, nidx, x, kpts, sd[p + ".offset_conv.weights"], extent) + sd[p + ".offset_bias"]
    dkp = off.view(-1, kpts.shape[0], 3) * extent + kpts
    kept = kp_kept(q_pts, s_pts, nidx, dkp, extent)
    if stats is not None:
        valid = (nidx >= 0) & (nidx < s_pts.shape[0])
        stats[p] = dict(kept=int(kept.sum()), dropped=int((valid & ~kept).sum()),
                        median_offset=float((dkp - kpts).norm(dim=-1).median()) / extent)
    return kp_conv(q_pts, s_pts, nidx, x, dkp, sd[p + ".weights"], extent, kept)


def kp_bn(x, sd, p, use_bn):
    return bn_eval(x, sd, p + ".batch_norm", KP_BN_EPS) if use_bn else x + sd[p + ".bias"]


def kp_unary(x, sd, p, use_bn, relu, slope):
    y = kp_bn(x @ sd[p + ".mlp.weight"].t(), sd, p + ".batch_norm", use_bn)
    return lrelu(y, slope) if relu else y


def kp_max_pool(x, idx):
    x = torch.cat([x, torch.zeros_like(x[:1])])
    return x[idx].max(dim=1)[0]


def kp_closest_pool(x, idx):
    x = torch.cat([x, torch.zeros_like(x[:1])])
    return x[idx[:, 0]]


def kpfcnn_plan(cfg):
    """Block plan mirroring KPFCNN.__init__ (kpconv.py:128-249): list of dicts."""
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
        enc.append(dict(kind=blk, radius=r, in_dim=in_dim, out_dim=out_dim, layer=layer,
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
        if "upsample" in blk:
            layer -= 1
            r *= 0.5
            out_dim //= 2
    return dict(encoder=enc, encoder_skips=skips, decoder=dec, decoder_concats=concats,
                head_in=out_dim)


def kpfcnn_forward(sd, batch, cfg, taps=None, stats=None):
    """batch: dict(features [N0,Cf], points[l] [N_l,3], neighbors[l] [N_l,H], pools[l], upsamples[l])
    -> logits [N0, C] (kpconv.py:270-291), with rigid and deformable blocks and either head.  stats collects
    kp_conv_deform's diagnostics per deformable conv."""
    plan = kpfcnn_plan(cfg)
    use_bn, slope = cfg.get("use_batch_norm", True), cfg.get("l_relu", 0.1)
    x = batch["features"]
    skip_x = []
    for bi, b in enumerate(plan["encoder"]):
        p = "encoder_blocks.%d" % bi
        if bi in plan["encoder_skips"]:
            skip_x.append(x)
        L = b["layer"]
        strided = "strided" in b["kind"]
        q = batch["points"][L + 1] if strided else batch["points"][L]
        s = batch["points"][L]
        nidx = batch["pools"][L] if strided else batch["neighbors"][L]

        def conv(y):
            if "deform" in b["kind"]:
                return kp_conv_deform(q, s, nidx, y, sd, p + ".KPConv", b["extent"], stats)
            return kp_conv(q, s, nidx, y, sd[p + ".KPConv.kernel_points"], sd[p + ".KPConv.weights"], b["extent"])
        if "simple" in b["kind"]:
            x = lrelu(kp_bn(conv(x), sd, p + ".batch_norm", use_bn), slope)
        elif "resnetb" in b["kind"]:
            feats = x
            y = feats
            if b["in_dim"] != b["out_dim"] // 4:
                y = kp_unary(y, sd, p + ".unary1", use_bn, True, slope)
            y = lrelu(kp_bn(conv(y), sd, p + ".batch_norm_conv", use_bn), slope)
            y = kp_unary(y, sd, p + ".unary2", use_bn, False, slope)
            sc = kp_max_pool(feats, nidx) if strided else feats
            if b["in_dim"] != b["out_dim"]:
                sc = kp_unary(sc, sd, p + ".unary_shortcut", use_bn, False, slope)
            x = lrelu(y + sc, slope)
        else:
            raise NotImplementedError(b["kind"])
        if taps is not None:
            taps[p] = x
    for bi, b in enumerate(plan["decoder"]):
        p = "decoder_blocks.%d" % bi
        if bi in plan["decoder_concats"]:
            x = torch.cat([x, skip_x.pop()], 1)
        if "upsample" in b["kind"]:
            x = kp_closest_pool(x, batch["upsamples"][b["layer"] - 1])
        elif b["kind"] == "unary":
            x = kp_unary(x, sd, p, use_bn, True, slope)
        else:
            raise NotImplementedError(b["kind"])
        if taps is not None:
            taps[p] = x
    if cfg.get("reduce_fc", False):
        # kpconv.py:229-240: head_mlp with BN (always) and LeakyReLU, head_softmax with a bias and no activation
        x = kp_unary(x, sd, "head_mlp", True, True, slope)
        return kp_unary(x, sd, "head_softmax", False, False, slope)
    # kpconv.py:241-251: both UnaryBlocks without BN and WITH LeakyReLU (no_relu keeps its default False on
    # head_softmax)
    x = kp_unary(x, sd, "head_mlp", False, True, slope)
    return kp_unary(x, sd, "head_softmax", False, True, slope)


def kp_batch_neighbors(queries, supports, q_lens, s_lens, radius, radius_search=None):
    """batch_neighbors (kpconv.py:2002-2034): dense [Nq,max] int, shadow = len(supports)."""
    radius_search = radius_search or O.c_radius
    qs = np.concatenate([[0], np.cumsum(q_lens)]).astype(np.int64)
    ss = np.concatenate([[0], np.cumsum(s_lens)]).astype(np.int64)
    idx, rs, _ = radius_search(supports, queries, radius, ss, qs)
    width = int((rs[1:] - rs[:-1]).max()) if len(rs) > 1 else 0
    return O.np_ragged_to_dense(idx, rs, width, np.int32(len(supports)))
