"""PointPillars at the nuScenes, Argoverse and Lyft configs: test support shared by tests/ref_pointpillars_configs.py
(which records tests/golden/pointpillars_config_<k>.npz), tests/test_oracle_pointpillars_configs.py,
tests/test_gpu_pointpillars_configs.py and bench_pointpillars_configs.py.

  * CONFIGS: the configs of the fixtures, the frames fed to them and their head-map shapes;
  * DETECT_CASES: the seeded head maps (detect_support.pp_detect_maps) the reference get_bboxes was recorded on;
  * synth_frame / load: the frames the reference's preprocess built, regenerated from their seeds and the recorded
    row mask and checked against the recorded digest, with the fixture's seeded weights and cfg;
  * pp_pfn / pointpillars_forward: the oracle forward of oracle/models_torch.py with a PillarFeatureNet of one or
    more PFNLayers (point_pillars.py:400-555); with one layer it is oracle/models_torch.pp_pfn itself.
Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
import hashlib
import json
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import models_torch as MT, weights
from open3d_ml_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# name -> (yml, frame seeds, points per frame, point channels, head map H = W)
CONFIGS = dict(
    nuscenes=dict(yml="pointpillars_nuscenes.yml", seeds=[31, 32], n=16000, channels=4, hw=200),
    argoverse=dict(yml="pointpillars_argoverse.yml", seeds=[41, 42], n=16000, channels=3, hw=200),
    lyft=dict(yml="pointpillars_lyft.yml", seeds=[51], n=24000, channels=4, hw=320),
)

# per head: a full-size map (so that the top-k cut decides) and a map with fewer rows than nms_pre and a class with
# nothing above score_thr
DETECT_CASES = [
    dict(name="nuscenes_full", head="nuscenes", H=200, W=200, seeds=[601], n_fg=1500, empty_classes=[]),
    dict(name="nuscenes_small", head="nuscenes", H=6, W=5, seeds=[602], n_fg=60, empty_classes=[3]),
    dict(name="argoverse_full", head="argoverse", H=200, W=200, seeds=[702], n_fg=1500, empty_classes=[]),
    dict(name="argoverse_small", head="argoverse", H=6, W=5, seeds=[702], n_fg=60, empty_classes=[1]),
    dict(name="lyft_full", head="lyft", H=320, W=320, seeds=[801], n_fg=1500, empty_classes=[]),
    dict(name="lyft_small", head="lyft", H=6, W=5, seeds=[802], n_fg=60, empty_classes=[5]),
]


def fixture(k):
    return os.path.join(GOLDEN, "pointpillars_config_%s.npz" % k)


def synth_frame(k, i, pc_range):
    """Frame i of config k as fed to the reference's preprocess: synth.lidar_frame in the config's range."""
    spec = CONFIGS[k]
    return synth.lidar_frame(spec["n"], spec["seeds"][i], tuple(pc_range), with_intensity=spec["channels"] == 4)


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def load(k):
    """(fixture, state_dict, cfg, frames) of config k.  The frames are the rows of synth_frame the reference's
    preprocess kept (the recorded mask), bit-equal to what its ConcatBatcher delivered (the recorded digest)."""
    g = np.load(fixture(k), allow_pickle=False)
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), int(g["weight_seed"]))
    cfg = json.loads(str(g["cfg"]))
    frames = []
    for i in range(int(g["frames"])):
        pts = synth_frame(k, i, cfg["point_cloud_range"])
        pts = pts[np.unpackbits(g["point_%d_kept" % i], count=len(pts)).astype(bool)]
        assert digest(pts) == str(g["point_%d_sha256" % i]), "frame %d of %s does not regenerate" % (i, k)
        frames.append(torch.from_numpy(pts))
    return g, sd, cfg, frames


def pfn_layer_count(sd):
    n = 0
    while "voxel_encoder.pfn_layers.%d.linear.weight" % n in sd:
        n += 1
    return n


def pp_pfn(pillars, counts, coords4, sd, cfg):
    """PillarFeatureNet with its PFNLayers -> [M, 64] (point_pillars.py:400-555).  Only the decorated input is
    masked: every slot, padded ones included, takes part in every layer's max, and a layer that is not the last
    passes cat(y[p], max over slots of y) on."""
    n = pfn_layer_count(sd)
    if n == 1:
        return MT.pp_pfn(pillars, counts, coords4, sd, cfg)
    vx, vy = cfg["voxel_size"][0], cfg["voxel_size"][1]
    x_off = vx / 2 + cfg["point_cloud_range"][0]
    y_off = vy / 2 + cfg["point_cloud_range"][1]
    cnt = counts.to(pillars.dtype).view(-1, 1, 1)
    mean = pillars[:, :, :3].sum(1, keepdim=True) / cnt
    f_center = torch.stack([
        pillars[:, :, 0] - (coords4[:, 3].to(pillars.dtype).unsqueeze(1) * vx + x_off),
        pillars[:, :, 1] - (coords4[:, 2].to(pillars.dtype).unsqueeze(1) * vy + y_off)], -1)
    f = torch.cat([pillars, pillars[:, :, :3] - mean, f_center], -1)
    slot = torch.arange(pillars.shape[1]).view(1, -1)
    f = f * (slot < counts.view(-1, 1)).unsqueeze(-1).to(f.dtype)
    for i in range(n):
        p = "voxel_encoder.pfn_layers.%d" % i
        y = torch.relu(MT.bn_eval(f @ sd[p + ".linear.weight"].t(), sd, p + ".norm", MT.PP_BN_EPS))
        m = y.max(dim=1, keepdim=True)[0]
        if i == n - 1:
            return m.squeeze(1)
        f = torch.cat([y, m.expand_as(y)], 2)


def pointpillars_forward(sd, frames, cfg, taps=None):
    """oracle/models_torch.pointpillars_forward with pp_pfn above: frames [N_i, C] -> (cls, reg, dir) NCHW."""
    pil, co, cn = [], [], []
    for b, pts in enumerate(frames):
        p, c, k = MT.pp_voxelize(pts, cfg)
        pil.append(p)
        co.append(F.pad(c, (1, 0), value=b))
        cn.append(k)
    pil, co, cn = torch.cat(pil), torch.cat(co), torch.cat(cn)
    vf = pp_pfn(pil, cn, co, sd, cfg)
    ny, nx = cfg["output_shape"]
    canvas = MT.pp_scatter(vf, co, len(frames), ny, nx)
    if taps is not None:
        taps.update(pillars=pil, coords=co, counts=cn, pfn=vf)
    return MT.pp_backbone_neck_head(canvas, sd, cfg)
