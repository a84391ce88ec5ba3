"""oracle/pvcnn.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The PVCNN oracle in one module: the float64 numpy rules of DESIGN.md section 2 (voxel coordinates and cells, average
voxelization, trilinear devoxelization), the margin nudge every parity input goes through, the plain-PyTorch port of
``PVCNN.forward`` (ml3d/torch/models/pvcnn.py:136-160; PVConv / Voxelization / avg_voxelize :559-664), functional and
driven by the reference's own ``state_dict`` keys like the ports of oracle/models_torch.py, and the binding that lets
the golden recorder run the unmodified reference class.

Grids are [B, X, Y, Z, C]: cell (x * r + y) * r + z of cloud b is row b * r^3 + (x * r + y) * r + z.
Only tests/, __graft_entry__.smoke() and bench_pvcnn.py may import this module.
"""
import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------- float64 rules
def np_pv_voxel_cells(coords, r, eps=1e-6):
    """coords [B, N, 3] -> (voxel coordinates float64 [B, N, 3] = clamp(((c - mean) / (2 max|c - mean| + eps) + 0.5) r,
    0, r - 1), global cell ids int64 [B, N] of their round-half-to-even)."""
    c = np.asarray(coords, np.float64)
    c = c - c.mean(1, keepdims=True)
    denom = 2.0 * np.sqrt((c * c).sum(2)).max(1) + eps
    v = np.clip((c / denom[:, None, None] + 0.5) * r, 0, r - 1)
    q = np.rint(v).astype(np.int64)
    cell = (q[..., 0] * r + q[..., 1]) * r + q[..., 2] + np.arange(len(c))[:, None] * r ** 3
    return v, cell


def np_avg_voxelize(feat, cell, num_cells):
    """feat [B, N, C], global cell ids [B, N] -> float64 [num_cells, C]: the mean over the points of a cell, 0 where
    there is none."""
    f = np.asarray(feat, np.float64).reshape(-1, np.shape(feat)[-1])
    ids = np.asarray(cell).reshape(-1)
    grid = np.zeros((num_cells, f.shape[1]))
    np.add.at(grid, ids, f)
    cnt = np.bincount(ids, minlength=num_cells)
    return grid / np.maximum(cnt, 1)[:, None]


def np_trilinear_devoxelize(vox, grid, r):
    """vox [B, N, 3] in [0, r - 1], grid [B, r^3, C] -> (outs [B, N, C], inds int32 [B, 8, N], wgts [B, 8, N]).  Per
    axis lo = floor(v), d = v - lo, hi = lo + (d > 0); corner k takes hi on x / y / z where bit 2 / 1 / 0 of k is
    set."""
    v = np.asarray(vox, np.float64)
    g = np.asarray(grid, np.float64)
    lo = np.floor(v)
    d = v - lo
    lo = lo.astype(np.int64)
    hi = lo + (d > 0)
    inds, wgts = [], []
    for k in range(8):
        bits = ((k >> 2) & 1, (k >> 1) & 1, k & 1)
        q = [hi[..., a] if b else lo[..., a] for a, b in enumerate(bits)]
        w = [d[..., a] if b else 1.0 - d[..., a] for a, b in enumerate(bits)]
        inds.append((q[0] * r + q[1]) * r + q[2])
        wgts.append(w[0] * w[1] * w[2])
    inds, wgts = np.stack(inds, 1), np.stack(wgts, 1)
    outs = sum(wgts[:, k, :, None] * np.take_along_axis(g, inds[:, k, :, None], 1) for k in range(8))
    return outs, inds.astype(np.int32), wgts


def pv_margin_nudge(points, resolutions, margin=1e-3, eps=1e-6):
    """`points` [N, 3] as float32 with every point whose float64 voxel coordinate lies within `margin` of a rounding
    boundary k + 0.5 at one of `resolutions` moved 2 * margin away from it, until none is left: float32 reductions in
    different orders then agree about every point's cell.  (Moving a point shifts the cloud's mean by 1 / N of the
    step, far less than the margin; dropping it would shift the mean by more than the margin.)"""
    p = np.array(points, np.float32)
    for _ in range(64):
        moved = False
        for r in resolutions:
            v = np_pv_voxel_cells(p[None], r, eps)[0][0]
            c = p.astype(np.float64) - p.astype(np.float64).mean(0)
            denom = 2.0 * np.sqrt((c * c).sum(1)).max() + eps
            frac = v - np.floor(v) - 0.5
            bad = np.abs(frac) < margin
            if bad.any():
                p[bad] += (np.where(frac >= 0, 2.0, -2.0) * margin * denom / r)[bad].astype(np.float32)
                moved = True
        if not moved:
            return p
    raise ValueError("pv_margin_nudge: did not settle")


# ------------------------------------------------------------------------------------------------- torch port
PV_BLOCKS = ((1, 32), (2, 16), (1, 16))    # PVCNN.blocks[:-1] as (repeats, resolution), pvcnn.py:83


def pv_voxel_coords(coords, r, eps=1e-6):
    """Voxelization.forward (pvcnn.py:653-661): coords [B, 3, N] -> clamped float voxel coordinates [B, 3, N]."""
    c = coords - coords.mean(2, keepdim=True)
    c = c / (c.norm(dim=1, keepdim=True).max(dim=2, keepdim=True).values * 2.0 + eps) + 0.5
    return torch.clamp(c * r, 0, r - 1)


def pv_avg_voxelize(feat, vox, r):
    """avg_voxelize (pvcnn.py:579-619): feat [B, C, N] -> [B, C, r, r, r], cell (x r + y) r + z of round(vox)."""
    B, C, N = feat.shape
    q = torch.round(vox).to(torch.int64)
    cell = ((q[:, 0] * r + q[:, 1]) * r + q[:, 2])[:, None, :]
    grid = torch.zeros((B, C, r ** 3), dtype=feat.dtype, device=feat.device).scatter_add_(2, cell.expand(-1, C, -1), feat)
    cnt = torch.zeros((B, 1, r ** 3), dtype=feat.dtype, device=feat.device).scatter_add_(
        2, cell, torch.ones_like(feat[:, :1]))
    return (grid / cnt.clamp(min=1)).view(B, C, r, r, r)


def pv_trilinear_devoxelize(resolution, is_training, coords, features):
    """open3d.ml.torch.ops.trilinear_devoxelize_forward by the rule of DESIGN.md section 2: coords [B, 3, N] in
    [0, r - 1], features [B, C, r, r, r] -> (outs [B, C, N], inds int32 [B, 8, N], wgts [B, 8, N])."""
    r = int(resolution)
    B, C = features.shape[:2]
    lo = torch.floor(coords)
    d = coords - lo
    lo = lo.to(torch.int64)
    hi = lo + (d > 0)
    g = features.reshape(B, C, r ** 3)
    inds, wgts, outs = [], [], 0
    for k in range(8):
        bits = ((k >> 2) & 1, (k >> 1) & 1, k & 1)
        q = [hi[:, a] if b else lo[:, a] for a, b in enumerate(bits)]
        w = [d[:, a] if b else 1 - d[:, a] for a, b in enumerate(bits)]
        inds.append((q[0] * r + q[1]) * r + q[2])
        wgts.append(w[0] * w[1] * w[2])
        outs = outs + wgts[k][:, None, :] * torch.gather(g, 2, inds[k][:, None, :].expand(-1, C, -1))
    return outs, torch.stack(inds, 1).to(torch.int32), torch.stack(wgts, 1)


def _pv_bn(x, sd, p, eps):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, eps)


def pv_shared_mlp(x, sd, p):
    """SharedMLP (pvcnn.py:455-501), one layer: Conv1d 1x1 + BatchNorm1d + ReLU over [B, C, N]."""
    return F.relu(_pv_bn(F.conv1d(x, sd[p + ".layers.0.weight"], sd[p + ".layers.0.bias"]), sd, p + ".layers.1", 1e-5))


def pvcnn_forward(sd, inputs, cfg, taps=None):
    """PVCNN.forward in eval mode.  inputs: point [B, 3, N], feat [B, C, N]; cfg: voxel_resolution_multiplier.
    -> logits [B, N, classes].  taps: "<block>.voxels" / ".conv0" / ".conv1" [B, C, r, r, r], "<block>" [B, N, C],
    "cloud_features" [B, C]."""
    coords, feat = inputs["point"], inputs["feat"]
    vr = cfg.get("voxel_resolution_multiplier", 1)
    res = [int(vr * r) for rep, r in PV_BLOCKS for _ in range(rep)]
    outs = []
    for i, r in enumerate(res):
        p = "point_features.%d" % i
        vox = pv_voxel_coords(coords, r)
        g = pv_avg_voxelize(feat, vox, r)
        if taps is not None:
            taps[p + ".voxels"] = g
        for j, li in enumerate((0, 3)):
            q = "%s.voxel_layers.%d" % (p, li)
            g = F.conv3d(g, sd[q + ".weight"], sd[q + ".bias"], padding=1)
            g = F.leaky_relu(_pv_bn(g, sd, "%s.voxel_layers.%d" % (p, li + 1), 1e-4), 0.1)
            if taps is not None:
                taps["%s.conv%d" % (p, j)] = g
        feat = pv_trilinear_devoxelize(r, False, vox, g)[0] + pv_shared_mlp(feat, sd, p + ".point_features")
        outs.append(feat)
        if taps is not None:
            taps[p] = feat.transpose(1, 2)
    feat = pv_shared_mlp(feat, sd, "point_features.%d" % len(res))
    outs.append(feat)
    cf = feat.max(dim=-1).values
    for j in (0, 1):
        p = "cloud_features.%d" % j
        cf = F.relu(_pv_bn(F.linear(cf, sd[p + ".0.weight"], sd[p + ".0.bias"]), sd, p + ".1", 1e-5))
    if taps is not None:
        taps["cloud_features"] = cf
    x = torch.cat(outs + [cf[:, :, None].expand(-1, -1, coords.shape[-1])], 1)
    x = pv_shared_mlp(x, sd, "classifier.0")
    x = pv_shared_mlp(x, sd, "classifier.2")
    return F.conv1d(x, sd["classifier.4.weight"], sd["classifier.4.bias"]).transpose(1, 2)


# ------------------------------------------------------------------------------------------- golden recorder
def bind_pvcnn_devoxelize():
    """For the golden recorder: the reference binds trilinear_devoxelize_forward only where it finds a CUDA device
    (pvcnn.py:13-14), so the oracle's rule goes into the imported module's globals; its source stays as it is."""
    from . import refshim
    refshim.install()
    import ml3d.torch.models.pvcnn as ref
    ref.trilinear_devoxelize_forward = pv_trilinear_devoxelize
    return ref
