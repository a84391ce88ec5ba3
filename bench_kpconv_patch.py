"""The reference KPFCNN forward before and after kpconv.patch_reference_model, on a batch as SemanticSegmentation
feeds it.

    python bench_kpconv_patch.py [--steps N] [--warmup W]

Needs the unmodified reference tree ($OPEN3D_ML_ROOT, or the oracle/_ref copy build() makes), bound through the shim.
Workload: the shipped kpconv_s3dis.yml model (seeded manifest weights, eval) with min_in_points = 5 000, so that the
pipeline's batch_size = 4 items fill its batch_limit of 20 000 points; each item is the reference's own preprocess /
transform of a synthetic 6 x 5 x 2.7 m room (synth.room_cloud, 60 000 points at 0.04 m), stacked by ConcatBatcher and
moved to the device.  The unpatched forward (the reference's eager torch layers on the GPU, torch's default float32
matmul precision) and the patched one are timed with CUDA events per call after warm-up, median over --steps, in three
alternating runs.
Prints one JSON line and writes nothing (the reference writes its kernel-point files into a temporary directory).
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_kpconv_deform import gpu_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kpconv_patch.py measures on a CUDA device; none is visible")
    from oracle.make_ref_snapshot import ref_root
    if ref_root() is None:
        raise SystemExit("bench_kpconv_patch.py runs the reference KPFCNN class: no reference tree or snapshot of it")
    import kpconv_patch_cases as C
    C.rbc.install("b200")
    os.chdir(tempfile.mkdtemp())
    import open3d.ml.torch as ml3d
    from open3d_ml_b200 import synth
    from open3d_ml_b200.kpconv import patch_reference_model
    torch.cuda.set_device(0)
    info = gpu_info()
    net, pipe_cfg = C.seeded_model(ref_root(), ("kpconv_s3dis.yml", dict(min_in_points=5000)))
    np.random.seed(0)
    pts, feats = synth.room_cloud(60000, 61)
    attr = {"split": "test"}
    data = net.preprocess({"point": pts, "feat": feats[:, 1:4] * 255, "label": np.zeros(len(pts), np.int32)}, attr)
    items = [{"data": net.transform(data, attr), "attr": attr} for _ in range(int(pipe_cfg["batch_size"]))]
    batch = ml3d.dataloaders.ConcatBatcher("cuda").collate_fn(items)["data"]
    net.to("cuda")
    net.device = "cuda"
    unpatched = net.forward
    patch_reference_model(net)
    patched = net.forward

    def call(fwd):
        with torch.no_grad():
            return fwd(batch)
    for _ in range(args.warmup):
        call(unpatched), call(patched)
    runs = []
    for _ in range(3):
        ref_ms, want = timed(lambda: call(unpatched), args.steps)
        fused_ms, got = timed(lambda: call(patched), args.steps)
        runs.append(dict(unpatched_ms=round(ref_ms, 3), patched_ms=round(fused_ms, 3)))
    print(json.dumps(dict(metric="reference KPFCNN forward, S3DIS config, unpatched vs patch_reference_model", gpu=info,
                          points=int(batch.points[0].shape[0]), items=len(batch.lengths[0]), runs=runs,
                          rel_err=float((got - want).abs().max() / want.abs().max()),
                          timed="CUDA events per call after %d warm-up calls of each: median of %d calls, three "
                                "alternating runs" % (args.warmup, args.steps))))


if __name__ == "__main__":
    main()
