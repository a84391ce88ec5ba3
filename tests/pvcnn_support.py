"""Builders of the PVCNN parity tests, shared with tests/golden/make_golden_pvcnn.py: seeded, margin-filtered inputs and the
two recorded reference cases."""
import json

import numpy as np
import torch

from oracle import pvcnn as PV, weights
from open3d_ml_b200 import synth
from open3d_ml_b200.pvcnn import block_resolutions

import helpers as H


def filtered_cloud(n, seed, resolutions):
    """(point [n, 3], feat [n, 9]) S3DIS-like rows none of which lies within 1e-3 of a rounding boundary at
    `resolutions`, so that reductions in different orders put every point in the same voxel.  The features keep the
    coordinates they were made from: only the voxelization needs the margin."""
    pts, feat = synth.pvcnn_s3dis_input(n, seed)
    return PV.pv_margin_nudge(pts, resolutions), feat


def pvcnn_inputs(B, N, seed0, cfg):
    """The reference's inputs dict: point [B, 3, N], feat [B, 9, N]."""
    res = sorted(set(block_resolutions(cfg)))
    clouds = [filtered_cloud(N, seed0 + b, res) for b in range(B)]
    return dict(point=torch.from_numpy(np.stack([c[0].T for c in clouds])).contiguous(),
                feat=torch.from_numpy(np.stack([c[1].T for c in clouds])).contiguous())


def recorded_case(tag):
    """-> (state_dict, cfg, inputs, fixture) of one case of boundary_pvcnn_class.npz ("shipped" or "odd")."""
    g = H.golden("boundary_pvcnn_class.npz")
    cfg = json.loads(str(g[tag + ".cfg"]))
    sd = weights.seeded_state_dict(json.loads(str(g[tag + ".manifest"])), int(g["weight_seed"]))
    return sd, cfg, pvcnn_inputs(int(g["B"]), int(g["N"]), cfg["seed0"], cfg), g


def check_recorded(g, tag, logits, taps, tol):
    """Sampled logits and taps of a forward against the fixture, each within tol of the recorded tensor's largest
    magnitude.  -> the largest relative error seen."""
    worst = 0.0
    want = g[tag + ".logits"]
    got = logits.detach().cpu().reshape(-1)[torch.from_numpy(g[tag + ".logits_idx"])].numpy()
    worst = max(worst, float(np.abs(got - want).max() / np.abs(want).max()))
    assert worst <= tol, ("logits", worst)
    for key in g.files:
        pre = tag + ".tap."
        if not key.startswith(pre) or key.endswith((".idx", ".max")):
            continue
        name = key[len(pre):]
        got = taps[name].detach().cpu().reshape(-1)[torch.from_numpy(g[key + ".idx"])].numpy()
        e = float(np.abs(got - g[key]).max() / float(g[key + ".max"]))
        assert e <= tol, (name, e)
        worst = max(worst, e)
    return worst


# Constructed cloud of the tie rule, at r = 4 and eps = 0: the mean is 0 and the largest norm 1 exactly, so x maps to
# 2 x + 2 and the others to 2.  (x, voxel coordinate, cell along x): 4 clamps to r - 1; 2.5, 1.5, 3.5 -> 3 (clamped),
# 0.5 round half to even.
TIE_R = 4
TIE_X = np.array([1.0, -1.0, 0.25, -0.25, 0.75, -0.75])
TIE_VOX_X = np.array([3.0, 0.0, 2.5, 1.5, 3.0, 0.5])
TIE_CELL_X = np.array([3, 0, 2, 2, 3, 0])


def tie_cloud():
    pts = np.zeros((1, len(TIE_X), 3), np.float32)
    pts[0, :, 0] = TIE_X
    return pts


def tie_cells():
    return (TIE_CELL_X * TIE_R + 2) * TIE_R + 2
