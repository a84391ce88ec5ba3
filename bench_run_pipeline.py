"""``pipeline.run_test()`` of the unmodified ``scripts/run_pipeline.py``, with the shim alone (the reference forwards) and
with the fused dispatch of ``python -m open3d_ml_b200.run_pipeline``.

    python bench_run_pipeline.py [--runs R]

Needs the unmodified reference tree ($OPEN3D_ML_ROOT, or the oracle/_ref copy build() makes).  Workload: the seeded
datasets of tests/run_pipeline_cases.py at the shipped configs' sizes (a 50 000-point SemanticKITTI scan for
RandLA-Net, 40 000-point S3DIS rooms for KPFCNN and PVCNN, a 60 000-point KITTI frame for PointPillars), run with
--split test and a seeded checkpoint.  Each run is a process of its own; inside it, a wrapper around run_test() takes
the wall time (ending in a device synchronise), and CUDA events in a forward pre-hook and post-hook sum the forward
time, first calls included (the fused build, graph capture and cold kernels fall there).  The remainder is the
dataloader, transform, batcher and inference_end.  RandLA-Net, KPFCNN and PointPillars alternate the shim-only and the
fused run R times; PVCNN, which the shim alone cannot run, is timed fused only.  SparseConvUnet is not timed: the
reference's run_test stops in its update_probs after the first forward.  Medians over the runs; prints one JSON line
and writes nothing under the repository (data, logs and results go to a temporary directory).
"""
import argparse
import json
import os
import runpy
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

COMPARED = ("randlanet_semantickitti", "kpconv_s3dis", "pointpillars_kitti")
FUSED_ONLY = ("pvcnn_s3dis",)


def child(mode, args):
    """One run_test() in this process; prints the timings."""
    import torch
    from open3d_ml_b200 import run_pipeline as RP
    script, rest = RP.prepare(args)
    if mode == "fused":
        from open3d_ml_b200.fuse import fuse_reference_models
        fuse_reference_models()
    import ml3d.torch.pipelines as P
    times = {}

    def wrap(cls):
        run_test = cls.run_test

        def timed_run_test(self):
            events = []
            pre = self.model.register_forward_pre_hook(
                lambda m, a: events.append([torch.cuda.Event(enable_timing=True)]) or events[-1][0].record())
            post = self.model.register_forward_hook(
                lambda m, a, o: events[-1].append(torch.cuda.Event(enable_timing=True)) or events[-1][1].record())
            torch.cuda.synchronize()
            t = time.perf_counter()
            run_test(self)
            torch.cuda.synchronize()
            times["wall_ms"] = (time.perf_counter() - t) * 1e3
            pre.remove()
            post.remove()
            times["forward_ms"] = sum(a.elapsed_time(b) for a, b in events)
            times["forwards"] = len(events)
        cls.run_test = timed_run_test
    wrap(P.SemanticSegmentation)
    wrap(P.ObjectDetection)
    sys.argv = [script] + rest
    try:
        runpy.run_path(script, run_name="__main__")
    except SystemExit as e:
        if e.code not in (None, 0):
            raise
    print("TIMES " + json.dumps(times), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_run_pipeline.py measures on a CUDA device; none is visible")
    from oracle.make_ref_snapshot import ref_root
    if ref_root() is None or not os.path.isfile(os.path.join(ref_root(), "scripts", "run_pipeline.py")):
        raise SystemExit("bench_run_pipeline.py runs the reference scripts/run_pipeline.py: no reference tree")
    from bench_kpconv_deform import gpu_info
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]), OPEN3D_ML_ROOT=ref_root())
    base = tempfile.mkdtemp()
    made = {}
    for fam in COMPARED + FUSED_ONLY:
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "run_pipeline_cases.py"), "make", fam,
                            os.path.join(base, fam)], capture_output=True, text=True, env=env, timeout=900)
        if r.returncode:
            raise SystemExit(r.stderr[-3000:])
        made[fam] = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])

    def once(fam, mode):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode] + made[fam]["args"],
                           cwd=os.path.join(base, fam), capture_output=True, text=True, env=env, timeout=1800)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("TIMES ")]
        if r.returncode or not lines:
            raise SystemExit("%s %s failed:\n%s" % (fam, mode, r.stderr[-3000:]))
        return json.loads(lines[-1][6:])

    samples = {}
    for _ in range(a.runs):
        for fam in COMPARED:
            for mode in ("shim", "fused"):
                samples.setdefault((fam, mode), []).append(once(fam, mode))
        for fam in FUSED_ONLY:
            samples.setdefault((fam, "fused"), []).append(once(fam, "fused"))
    out = {}
    for (fam, mode), ts in samples.items():
        wall = statistics.median(t["wall_ms"] for t in ts)
        fwd = statistics.median(t["forward_ms"] for t in ts)
        out.setdefault(fam, {})[mode] = dict(wall_ms=round(wall, 1), forward_ms=round(fwd, 1),
                                             remainder_ms=round(wall - fwd, 1), forwards=ts[0]["forwards"])
    print(json.dumps(dict(metric="run_pipeline.py --split test: run_test() wall, summed forward and remainder (ms), "
                          "median of %d runs" % a.runs, gpu=gpu_info(), results=out)))


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3:])
    else:
        main()
