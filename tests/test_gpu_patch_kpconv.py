"""kpconv.patch_reference_model: the UNMODIFIED reference KPFCNN class running its forward on the fused path, driven by
the reference's own preprocess / transform / ConcatBatcher and SemanticSegmentation pipeline through the shim.  Every
case runs in one process of its own (tests/kpconv_patch_cases.py; the shim owns sys.modules['open3d']).

The module sorts after test_gpu_launch_count.py on purpose, so that the profiler-based modules run at the same point of
the pytest process as they did before it existed: on some hosts torch.profiler drops the kernel records of whole
sessions for stretches of a process (the kernels are timestamped outside the session's window), so their outcome
depends on when they run, and these cases take about a minute."""
import json
import os
import subprocess
import sys

import pytest

from oracle.make_ref_snapshot import ref_root

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(ref_root() is None, reason="no reference tree or snapshot of it")]
TOL = 1e-4
HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ("parity_s3dis", "parity_parislille3d", "flow", "refusals")


@pytest.fixture(scope="module")
def results():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(HERE), HERE]))
    r = subprocess.run([sys.executable, os.path.join(HERE, "kpconv_patch_cases.py"), *CASES], capture_output=True,
                       text=True, timeout=1200, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    out = [json.loads(ln[len("RESULT "):]) for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
    assert all(res["device"] == "cuda" for res in out), out
    return {res["case"]: res for res in out}


@pytest.mark.parametrize("case,classes,deformable", [("parity_s3dis", 13, False), ("parity_parislille3d", 9, True)])
def test_patched_forward_matches_the_unpatched_class_on_the_gpu(results, case, classes, deformable):
    """The S3DIS config (rigid) and the Paris-Lille3D one (deformable layers, reduce_fc head), on one batch of the
    reference batcher with int64 indices, passed both as the batcher left it (host) and after KPConvBatch.to(cuda)."""
    res = results[case]
    n = res["levels"][0]
    assert res["ref_shape"] == [n, classes] and n >= 4000, res
    assert res["index_dtypes"] == ["torch.int64"]
    assert bool(res["deform_blocks"]) == deformable
    assert res["fused_shape"] == [n, classes] and res["fused_dtype"] == "torch.float32"
    assert res["fused_device"] == "cuda"
    assert res["rel_err"] < TOL and res["rel_err_host_batch"] < TOL, res


def test_run_inference_with_the_patched_model(results):
    """SemanticSegmentation.run_inference with the shipped S3DIS config: several batches of changing size, then
    predictions of the input's length that agree with the unpatched run from the same seeds."""
    res = results["flow"]
    n = res["n"]
    assert res["fused_labels_shape"] == [n] and res["fused_scores_shape"] == [n, 13], res
    assert res["labels_shape"] == [n] and res["scores_shape"] == [n, 13]
    assert res["fused_batch_points"] == res["batch_points"] and len(set(res["batch_points"])) > 1, res
    assert res["fused_finite"]
    assert res["label_agreement"] > 0.99 and res["score_max_diff"] < 1e-2, res


def test_refusals_and_state_dict_after_patching(results):
    res = results["refusals"]
    assert "inference-only" in (res["train_error"] or ""), res
    assert res["keys_unchanged"] and res["forward_still_patched"], res
    assert "modulated" in (res["modulated_error"] or ""), res
    assert res["modulated_forward_untouched"], res
