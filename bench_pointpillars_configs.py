"""PointPillars at each shipped config of the reference: KITTI, Waymo, Lyft (one-layer pillar feature net) and nuScenes,
Argoverse (two-layer).

    python bench_pointpillars_configs.py [--frames B] [--reps R]

Per config: the fused forward (voxelize + pillar feature net + scatter eagerly, backbone / neck / head as one CUDA
graph replay), the pillar feature net + scatter launch alone, and get_bboxes_padded on the forward's head maps, each
timed with CUDA events in steady state; plus the pillars and kept points of the batch.  Weights are seeded from the
manifests of tests/golden/ (KITTI, Waymo: pointpillars_<k>.manifest.json with the head of
boundary_pointpillars_detect.npz; the others: pointpillars_config_<k>.npz, which holds cfg_from_reference of the yml).
Frames are synth.lidar_frame in the config's range with its point channels (seeds 1000 + b).  Prints one JSON line
with the card's name, power limit and max SM clock, and writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

# points per frame: about a KITTI / nuScenes / Argoverse sweep, a Waymo frame, a Lyft sweep
POINTS = dict(kitti=20000, waymo=180000, lyft=60000, nuscenes=35000, argoverse=35000)


def ev_time_ms(fn, reps, warm):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def model(k):
    """(state_dict, cfg, point channels) of config k."""
    from oracle import weights
    golden = os.path.join(ROOT, "tests", "golden")
    if k in ("kitti", "waymo"):
        man, extra = weights.load_manifest(os.path.join(golden, "pointpillars_%s.manifest.json" % k))
        head = json.loads(str(np.load(os.path.join(golden, "boundary_pointpillars_detect.npz"))["cfg_" + k]))
        return weights.seeded_state_dict(man, 1), dict(extra["cfg"], head=head["head"],
                                                       num_classes=head["num_classes"]), 4
    from pp_configs_support import CONFIGS, fixture
    g = np.load(fixture(k))
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), int(g["weight_seed"]))
    return sd, json.loads(str(g["cfg"])), CONFIGS[k]["channels"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import open3d_ml_b200 as M
    from open3d_ml_b200 import synth
    torch.cuda.set_device(0)
    res = {}
    for k in ("kitti", "waymo", "lyft", "nuscenes", "argoverse"):
        sd, cfg, ch = model(k)
        net = M.PointPillarsB200(sd, cfg)
        frames = [torch.from_numpy(synth.lidar_frame(POINTS[k], 1000 + b, tuple(cfg["point_cloud_range"]),
                                                     with_intensity=ch == 4)).cuda() for b in range(args.frames)]
        fwd_ms = ev_time_ms(lambda: net(frames), args.reps, 5)
        canvas, vox = net.front_end(frames)
        pfn_ms = ev_time_ms(lambda: net.pfn_scatter(vox, canvas), args.reps, 5)
        cls, reg, dir_ = net(frames)
        det_ms = ev_time_ms(lambda: net.get_bboxes_padded(cls, reg, dir_), args.reps, 5)
        pillars, points = vox["counts"].tolist()
        res[k] = dict(pfn_layers=net.pfn_layers, points=POINTS[k] * args.frames, pillars=int(pillars),
                      kept_points=int(points), map_hw=[int(cls.shape[2]), int(cls.shape[3])],
                      forward_ms=round(fwd_ms, 4), pfn_scatter_ms=round(pfn_ms, 4), get_bboxes_padded_ms=round(det_ms, 4),
                      boxes=net.get_bboxes_padded(cls, reg, dir_)[3].tolist())
    print(json.dumps(dict(metric="PointPillars per config", frames=args.frames, configs=res, gpu=gpu_info(),
                          timed="CUDA events, steady state, x%d each after 5 warm-up calls" % args.reps)))


if __name__ == "__main__":
    main()
