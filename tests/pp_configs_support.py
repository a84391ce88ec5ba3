"""PointPillars at the nuScenes, Argoverse and Lyft configs: test support shared by tests/ref_pointpillars_configs.py
(which records tests/golden/pointpillars_config_<k>.npz), tests/test_oracle_pointpillars_configs.py,
tests/test_gpu_pointpillars_configs.py and bench_pointpillars_configs.py.

  * CONFIGS: the configs of the fixtures, the frames fed to them and their head-map shapes;
  * DETECT_CASES: the seeded head maps (detect_support.pp_detect_maps) the reference get_bboxes was recorded on;
  * synth_frame / load: the frames the reference's preprocess built, regenerated from their seeds and the recorded
    row mask and checked against the recorded digest, with the fixture's seeded weights and cfg.
The forward the fixtures pin is oracle/models_torch.pointpillars_forward, which runs one- and two-layer PFNs alike.
Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
import hashlib
import json
import os

import numpy as np
import torch

from oracle import weights
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

