"""The launcher's refusals, and that nothing is wrapped without ``fuse_reference_models()``.  No CUDA call: every case
runs in a process of its own (the shim owns sys.modules['open3d'])."""
import os
import subprocess
import sys

import pytest

from oracle.make_ref_snapshot import ref_root

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
needs_ref = pytest.mark.skipif(ref_root() is None or not os.path.isfile(
    os.path.join(ref_root() or "", "scripts", "run_pipeline.py")), reason="no reference tree or snapshot of it")


def _launch(args, env=None, cwd=None):
    e = dict(os.environ, PYTHONPATH=REPO, CUDA_VISIBLE_DEVICES="")
    e.pop("OPEN3D_ML_ROOT", None)
    e.update(env or {})
    return subprocess.run([sys.executable, "-m", "open3d_ml_b200.run_pipeline"] + args, capture_output=True,
                          text=True, timeout=300, env=e, cwd=cwd or REPO)


def test_no_root_is_refused(tmp_path):
    r = _launch(["torch", "-c", "x.yml", "--split", "test"], cwd=str(tmp_path))
    assert r.returncode != 0 and "no Open3D-ML tree" in r.stderr, r.stderr[-2000:]
    r = _launch(["--ml3d-root", str(tmp_path), "torch", "--split", "test"], cwd=str(tmp_path))
    assert r.returncode != 0 and "is not an Open3D-ML tree" in r.stderr, r.stderr[-2000:]


@needs_ref
@pytest.mark.parametrize("args,message", [
    (["tf", "-c", "x.yml", "--split", "test"], "runs the torch models only"),
    (["torch", "-c", "x.yml", "--split", "test", "--device_ids", "0", "1"], "distributed runs"),
])
def test_tf_and_distributed_runs_are_refused_before_the_script_runs(tmp_path, args, message):
    # the script would print "regular arguments" as its first act, and fail on the missing config after it
    r = _launch(["--ml3d-root", ref_root()] + args, cwd=str(tmp_path))
    assert r.returncode != 0 and message in r.stderr, r.stderr[-2000:]
    assert "regular arguments" not in r.stdout


@needs_ref
def test_the_shim_alone_leaves_the_reference_classes_unwrapped():
    code = ("import sys; sys.path.insert(0, %r); import open3d_ml_b200; from open3d_ml_b200 import shim, fuse;"
            "shim.install(%r); import open3d.ml.torch as ml3d; c = fuse.reference_classes();"
            "assert sorted(c) == ['KPFCNN', 'PVCNN', 'PointPillars', 'RandLANet', 'SparseConvUnet'];"
            "assert not any(fuse.is_fused(k) for k in c.values()), c;"
            "fuse.fuse_reference_models(); fuse.fuse_reference_models();"
            "assert all(fuse.is_fused(k) and not fuse.is_fused(type('X', (), {'forward': k.forward.__wrapped__}))"
            " for k in c.values()); print('ok')" % (REPO, ref_root()))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-3000:]
