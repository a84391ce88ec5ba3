"""``python -m open3d_ml_b200.run_pipeline``: the UNMODIFIED reference ``scripts/run_pipeline.py --split test`` on the
five shipped model families, on seeded on-disk datasets with a checkpoint that the pipeline loads after
``model.eval()`` (tests/run_pipeline_cases.py).  Every run is a process of its own (the shim owns
sys.modules['open3d']); they run four at a time."""
import glob
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle.make_ref_snapshot import ref_root

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(ref_root() is None or not os.path.isfile(
    os.path.join(ref_root() or "", "scripts", "run_pipeline.py")), reason="no reference tree or snapshot of it")]
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
CASES = os.path.join(HERE, "run_pipeline_cases.py")
FAMILIES = ("randlanet_semantickitti", "kpconv_s3dis", "pointpillars_kitti", "pvcnn_s3dis", "sparseconvunet_scannet")
CLASS = dict(randlanet_semantickitti="RandLANet", kpconv_s3dis="KPFCNN", pointpillars_kitti="PointPillars",
             pvcnn_s3dis="PVCNN", sparseconvunet_scannet="SparseConvUnet")
COMPARED = ("randlanet_semantickitti", "kpconv_s3dis", "pointpillars_kitti")


def _env():
    return dict(os.environ, PYTHONPATH=os.pathsep.join([REPO, HERE]), OPEN3D_ML_ROOT=ref_root())


def _run(cmd, cwd):
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=1800, env=_env())
    return dict(rc=r.returncode, out=r.stdout, err=r.stderr)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    base = tmp_path_factory.mktemp("run_pipeline")
    made = {}
    for fam in FAMILIES:
        r = subprocess.run([sys.executable, CASES, "make", fam, str(base / fam)], capture_output=True, text=True,
                           timeout=900, env=_env())
        assert r.returncode == 0, r.stderr[-3000:]
        made[fam] = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
    jobs = {}
    for fam, m in made.items():
        d = str(base / fam)
        jobs[(fam, "module")] = ([sys.executable, "-m", "open3d_ml_b200.run_pipeline"] + m["args"], d)
        modes = ["shim"] + (["launch"] if fam in COMPARED else []) + (
            ["patched", "stale"] if fam == "randlanet_semantickitti" else [])
        for mode in modes:
            jobs[(fam, mode)] = ([sys.executable, CASES, "run", mode, os.path.join(d, "out_" + mode), "--"]
                                 + m["args"], d)
    with ThreadPoolExecutor(4) as ex:
        futs = {k: ex.submit(_run, *v) for k, v in jobs.items()}
        res = {k: f.result() for k, f in futs.items()}
    for (fam, mode), r in res.items():
        r["made"] = made[fam]
        r["out_dir"] = os.path.join(str(base / fam), "out_" + mode)
    return res


def _saved(fam, test):
    """What save_test_result wrote: {name: number of points (segmentation) or 1 (a KITTI frame's box file)}."""
    if fam == "randlanet_semantickitti":
        return {"11_" + os.path.basename(f)[:-6]: os.path.getsize(f) // 4
                for f in glob.glob(os.path.join(test, "sequences", "11", "predictions", "*.label"))}
    if fam == "pointpillars_kitti":
        return {os.path.basename(f)[:-4]: 1 for f in glob.glob(os.path.join(test, "*.txt"))}
    return {os.path.basename(f)[:-4]: len(np.load(f)) for f in glob.glob(os.path.join(test, "*", "*.npy"))}


@pytest.mark.parametrize("fam", FAMILIES)
def test_every_family_runs_the_unmodified_script_through_the_launcher(runs, fam):
    r = runs[(fam, "module")]
    if fam == "sparseconvunet_scannet":
        # the fused forward runs; then SemanticSegmentation.update_tests calls SparseConvUnet.update_probs with three
        # arguments where the reference declares four, which stops the reference's own run_test after the first batch
        assert r["rc"] != 0 and "update_probs() missing 1 required positional argument" in r["err"], r["err"][-3000:]
        assert "open3d_ml_b200: SparseConvUnet runs its fused forward" in r["err"]
        return
    assert r["rc"] == 0, r["err"][-4000:]
    if fam == "pointpillars_kitti":
        # ObjectDetectBatch leaves its attr list empty, so KITTI.save_test_result writes no file; the boxes of every
        # frame are checked from what save_test_result received (test_launcher_agrees_with_the_reference_forward)
        assert _saved(fam, r["made"]["test"]) == {}
    else:
        assert _saved(fam, r["made"]["test"]) == r["made"]["expect"]
    assert "open3d_ml_b200: %s runs its fused forward" % CLASS[fam] in r["err"], r["err"][-2000:]


@pytest.mark.parametrize("fam,error", [("pvcnn_s3dis", "NameError"), ("sparseconvunet_scannet", "voxel")])
def test_the_shim_alone_cannot_run_pvcnn_and_sparseconvunet(runs, fam, error):
    r = runs[(fam, "shim")]
    assert r["rc"] != 0
    tail = r["err"][-3000:]
    assert error in tail.splitlines()[-1] if error == "NameError" else error in tail, tail


def _load(d):
    return {os.path.basename(f)[:-4]: dict(np.load(f, allow_pickle=False)) for f in glob.glob(os.path.join(d, "*.npz"))}


@pytest.mark.parametrize("fam", COMPARED)
def test_launcher_agrees_with_the_reference_forward(runs, fam):
    """Same command, same seeds: the fused dispatch against the reference forward under the shim alone."""
    fused, ref = runs[(fam, "launch")], runs[(fam, "shim")]
    assert fused["rc"] == 0 and ref["rc"] == 0, (fused["err"][-3000:], ref["err"][-3000:])
    a, b = _load(fused["out_dir"]), _load(ref["out_dir"])
    assert sorted(a) == sorted(fused["made"]["expect"]) == sorted(b)
    for name in a:
        if fam == "pointpillars_kitti":
            x, y = a[name]["boxes"], b[name]["boxes"]      # rows: centre, size, yaw, confidence
            assert x.shape == y.shape and len(x) > 0, (name, x.shape, y.shape)
            # the seeded weights leave hundreds of overlapping boxes of close scores per frame, so the boxes are not
            # paired one to one: the same count, the same classes and the same sorted confidences, to the score
            # bound of the segmentation models
            assert sorted(a[name]["labels"]) == sorted(b[name]["labels"])
            assert np.allclose(np.sort(x[:, 7]), np.sort(y[:, 7]), atol=1e-2)
        else:
            assert (a[name]["labels"] == b[name]["labels"]).mean() > 0.99
            assert float(np.abs(a[name]["scores"] - b[name]["scores"]).max()) < 1e-2


def test_the_checkpoint_loaded_after_eval_is_the_one_that_runs(runs):
    """run_test calls model.eval() and only then load_ckpt: the launcher's predictions are those of the model patched
    after the checkpoint loaded, not those of the weights it held at eval()."""
    fam = "randlanet_semantickitti"
    for mode in ("launch", "patched", "stale"):
        assert runs[(fam, mode)]["rc"] == 0, runs[(fam, mode)]["err"][-3000:]
    got, want, stale = (_load(runs[(fam, m)]["out_dir"]) for m in ("launch", "patched", "stale"))
    for name in got:
        assert (got[name]["labels"] == want[name]["labels"]).mean() > 0.999
        assert float(np.abs(got[name]["scores"] - want[name]["scores"]).max()) < 1e-3
        assert float(np.abs(got[name]["scores"] - stale[name]["scores"]).max()) > 0.05
