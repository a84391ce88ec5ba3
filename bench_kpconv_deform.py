"""Deformable KPConv benchmark: KPFCNNB200 on the Paris-Lille3D config (deformable layers 2-4) against the torch port
run eagerly on the same GPU.

    python bench_kpconv_deform.py [--steps N] [--warmup W]

Workload: 4 m spheres cropped from synthetic LiDAR frames (synth.semantickitti_cloud), grid-subsampled at 0.08 m and
stacked to batch_limit = 20 000 points (tests/helpers.paris_clouds, seed 1000); the batch is built on the device by
kpconv.build_batch with the deform radii of kpconv.layer_radii.  Weights: the manifest of
tests/golden/boundary_kpconv_deform_class.npz, seed 1.  The fused forward is timed with CUDA events per step after
warm-up (median over --steps), in two runs alternating with the eager port (oracle/models_torch.kpfcnn_forward,
median over --steps / 10).  For every deformable KPConv it reports H (neighbour row width), the fraction of valid
neighbours the re-selection keeps, and the median time of its four steps: offset gather (rigid kpconv_gather), offset
GEMM, deformable gather, GEMM + BN + LeakyReLU.  Prints one JSON line and writes nothing.
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


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in out[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def timed(fn, steps):
    """-> (median ms per call, the last result) with one event pair per call."""
    ms, out = [], None
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kpconv_deform.py measures on a CUDA device; none is visible")
    import open3d_ml_b200 as M
    from open3d_ml_b200.kpconv import build_batch
    from oracle import models_torch as MT, weights
    from helpers import paris_clouds
    torch.cuda.set_device(0)
    info = gpu_info()
    g = np.load(os.path.join(ROOT, "tests", "golden", "boundary_kpconv_deform_class.npz"))
    cfg = json.loads(str(g["cfg"]))
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), 1)
    clouds = paris_clouds(1000)
    batch = build_batch(clouds, cfg)
    net = M.KPFCNNB200(sd, cfg)
    sdc = {k: v.cuda() for k, v in sd.items()}

    def port():
        with torch.no_grad():
            return MT.kpfcnn_forward(sdc, batch, cfg)
    for _ in range(args.warmup):
        net(batch)
    port()
    runs = []
    for _ in range(2):
        fused_ms, got = timed(lambda: net(batch), args.steps)
        port_ms, want = timed(port, max(3, args.steps // 10))
        runs.append(dict(fused_ms=round(fused_ms, 3), gpu_eager_port_ms=round(port_ms, 3)))
    rel = float((got - want).abs().max() / want.abs().max())

    per = {}
    for _ in range(args.steps):
        probe = []
        net(batch, probe=probe)
        torch.cuda.synchronize()
        for c in probe:
            e = c["events"]
            per.setdefault(c["name"], []).append([e[i].elapsed_time(e[i + 1]) for i in range(4)])
    convs = []
    for c in probe:
        dkp = c["offsets"].view(-1, c["kernel_points"].shape[0], 3) * c["extent"] + c["kernel_points"]
        kept = MT.kp_kept(c["q_pts"], c["s_pts"], c["neighbors"], dkp, c["extent"])
        valid = (c["neighbors"] >= 0) & (c["neighbors"] < c["s_pts"].shape[0])
        med = np.median(np.array(per[c["name"]]), axis=0)
        convs.append(dict(conv=c["name"], queries=int(c["q_pts"].shape[0]), H=int(c["neighbors"].shape[1]),
                          kept_fraction=round(float(kept.sum()) / max(1, int(valid.sum())), 4),
                          step_ms=dict(offset_gather=round(float(med[0]), 4), offset_gemm=round(float(med[1]), 4),
                                       deform_gather=round(float(med[2]), 4), gemm=round(float(med[3]), 4))))
    print(json.dumps(dict(metric="KPFCNN Paris-Lille3D forward (deformable layers 2-4)", gpu=info,
                          points=int(batch["points"][0].shape[0]), clouds=len(clouds), runs=runs,
                          fused_vs_port_rel_err=rel, deformable_convs=convs,
                          timed="CUDA events per step after %d warm-up steps: median of %d fused steps and %d port "
                                "steps, two alternating runs" % (args.warmup, args.steps, max(3, args.steps // 10)))))


if __name__ == "__main__":
    main()
