"""PointPillars box decoding benchmark: the fused PointPillarsB200.get_bboxes_padded (detect.cu) against the reference
flow restated in eager torch on the same GPU.

    python bench_detect.py [--shape kitti|waymo] [--frames B] [--reps R]

The head maps come from one fused forward of bench.py's PointPillars workload: the same manifest, seeded weights
(seed 1) and synthetic frames (seeds 1000 + b); one KITTI frame by default, 32 Waymo-shaped frames with
`--shape waymo`.  The head cfg (nms_pre, score_thr, dir_offset, anchors) is the reference yml's, as recorded in
tests/golden/boundary_pointpillars_detect.npz.  The reference arm is tests/detect_support.pp_get_bboxes with the
library's `nms` op: per frame and class the boolean-mask selects and the op's count read-back of
Anchor3DHead.get_bboxes / multiclass_nms.  Both are timed with CUDA events in steady state.  Prints one JSON line and
writes nothing.
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
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:  # noqa: BLE001
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="kitti", choices=["kitti", "waymo"])
    ap.add_argument("--frames", type=int, default=0, help="frames in the batch (0: 1 for kitti, 32 for waymo)")
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import open3d_ml_b200 as M
    from open3d_ml_b200 import synth
    from oracle import weights
    from detect_support import pp_get_bboxes
    torch.cuda.set_device(0)
    B = args.frames or (32 if args.shape == "waymo" else 1)
    man, extra = weights.load_manifest(os.path.join(ROOT, "tests", "golden", "pointpillars_%s.manifest.json" % args.shape))
    g = np.load(os.path.join(ROOT, "tests", "golden", "boundary_pointpillars_detect.npz"))
    head = json.loads(str(g["cfg_" + args.shape]))
    cfg = dict(extra["cfg"], head=head["head"], num_classes=head["num_classes"])
    net = M.PointPillarsB200(weights.seeded_state_dict(man, 1), cfg)
    if args.shape == "waymo":
        frames = [synth.lidar_frame(180000, 1000 + b, (-74.88, -74.88, -2, 74.88, 74.88, 4)) for b in range(B)]
    else:
        frames = [synth.lidar_frame(20000, 1000 + b) for b in range(B)]
    cls, reg, dir_ = net([torch.from_numpy(f).cuda() for f in frames])
    h = cfg["head"]
    fused_ms = ev_time_ms(lambda: net.get_bboxes_padded(cls, reg, dir_), args.reps, 5)
    counts = net.get_bboxes_padded(cls, reg, dir_)[3].tolist()
    anchors = net.anchors(cls.shape[2], cls.shape[3], cls.device)
    ref_ms = ev_time_ms(lambda: pp_get_bboxes(cls, reg, dir_, anchors, cfg["num_classes"], h["nms_pre"], h["score_thr"],
                                              h["dir_offset"], nms=M.nms, with_margins=False),
                        max(3, args.reps // 10), 2)
    print(json.dumps(dict(metric="PointPillars box decoding", shape=args.shape, frames=B,
                          map_hw=[int(cls.shape[2]), int(cls.shape[3])], nms_pre=h["nms_pre"],
                          fused_ms=round(fused_ms, 4), reference_ms=round(ref_ms, 4), boxes_per_frame=counts,
                          gpu=gpu_info(),
                          timed="CUDA events, steady state: get_bboxes_padded x%d / the eager torch flow x%d"
                                % (args.reps, max(3, args.reps // 10)))))


if __name__ == "__main__":
    main()
