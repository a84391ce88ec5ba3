"""fuse.fuse_reference_models(): the dispatch between the fused and the reference forward of unmodified reference
instances, and how it follows their weights (tests/fuse_cases.py, in one process of its own)."""
import json
import os
import subprocess
import sys

import pytest

from oracle.make_ref_snapshot import ref_root

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(ref_root() is None, reason="no reference tree or snapshot of it")]
HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1e-4


@pytest.fixture(scope="module")
def res():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(HERE), HERE]))
    r = subprocess.run([sys.executable, os.path.join(HERE, "fuse_cases.py")], capture_output=True, text=True,
                       timeout=1200, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


def test_train_mode_runs_the_reference_forward_bit_for_bit(res):
    r = res["randlanet"]
    assert r["train_bits_equal"] and r["train_builds"] == 0, r


def test_eval_mode_runs_the_fused_forward_and_builds_it_once(res):
    r = res["randlanet"]
    assert r["eval_builds_after_two_calls"] == 1 and r["eval_repeat_equal"], r
    assert r["eval_vs_fresh_fused"] == 0.0 and r["eval_vs_reference"] < TOL, r


def test_load_state_dict_between_two_eval_calls_rebuilds(res):
    r = res["randlanet"]
    # builds: the first eval call, the fresh fused model of the test, the rebuild after load_state_dict
    assert r["builds_after_load_state_dict"] == 3, r
    assert r["second_vs_fresh_fused"] == 0.0 and r["second_vs_first"] > 1e-2, r


def test_a_refused_config_warns_once_and_runs_the_reference_forward(res):
    assert res["kpconv"]["refused_equal_reference"], res["kpconv"]
    warnings = [m for lvl, m in res["log"] if lvl == "WARNING"]
    assert len(warnings) == 1 and "KPFCNN" in warnings[0] and "modulated" in warnings[0], res["log"]
    infos = [m for lvl, m in res["log"] if lvl == "INFO"]
    assert sorted(infos) == ["open3d_ml_b200: PointPillars runs its fused forward",
                             "open3d_ml_b200: RandLANet runs its fused forward"], res["log"]


def test_pointpillars_get_bboxes_follows_the_mode(res):
    r = res["pointpillars"]
    assert r["eval_fused_decode"] and r["train_reference_decode"], r
