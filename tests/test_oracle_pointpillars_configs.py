"""The oracle forward with a PillarFeatureNet of one or two layers (oracle/models_torch.pointpillars_forward) and the
oracle box decoding (detect_support.pp_get_bboxes) against the UNMODIFIED reference PointPillars built from its
nuScenes, Argoverse and Lyft ymls, recorded in tests/golden/pointpillars_config_<k>.npz
(`python tests/ref_pointpillars_configs.py --ops oracle --record tests/golden`).  Runs without a GPU."""
import json

import numpy as np
import pytest
import torch

from detect_support import pp_detect_maps, pp_get_bboxes
from open3d_ml_b200.pointpillars import grid_anchors
from oracle.models_torch import pointpillars_forward
from pp_configs_support import CONFIGS, DETECT_CASES, fixture, load
from test_oracle_detect import assert_margins

TOL = 2e-5  # float32 re-association between two CPU implementations, relative to the output's max |value|

# linear weight shapes of each config's PillarFeatureNet and its head maps' channels (cls, reg, dir)
SHAPES = dict(nuscenes=([[32, 9], [64, 64]], [98, 98, 28]), argoverse=([[32, 8], [64, 64]], [50, 70, 20]),
              lyft=([[64, 9]], [162, 126, 36]))


def sampled_rel_err(got, g, name):
    assert list(got.shape) == g[name + "_shape"].tolist()
    a = got.detach().double().reshape(-1)[torch.from_numpy(g[name + "_idx"])]
    return float((a - torch.from_numpy(g[name + "_val"])).abs().max() / float(g[name + "_absmax"]))


@pytest.mark.parametrize("k", list(CONFIGS))
def test_oracle_forward_matches_reference_fixture(k):
    g, sd, cfg, frames = load(k)
    pfn, heads = SHAPES[k]
    assert [list(sd["voxel_encoder.pfn_layers.%d.linear.weight" % i].shape) for i in range(len(pfn))] == pfn
    assert "voxel_encoder.pfn_layers.%d.linear.weight" % len(pfn) not in sd
    assert cfg["max_num_points"] == 20 and cfg["head"]["nms_pre"] == 1000
    assert all(f.shape[1] == CONFIGS[k]["channels"] for f in frames)
    taps = {}
    with torch.no_grad():
        outs = pointpillars_forward(sd, frames, cfg, taps=taps)
    hw = CONFIGS[k]["hw"]
    assert [list(o.shape) for o in outs] == [[len(frames), c, hw, hw] for c in heads]
    errs = [sampled_rel_err(o, g, "ref_%d" % i) for i, o in enumerate(outs)]
    assert all(e < TOL for e in errs), errs
    # nearly every real pillar has fewer points than slots: the padded slots are part of the comparison
    assert float((taps["counts"] < cfg["max_num_points"]).float().mean()) > 0.5


def head_fixture(case):
    return np.load(fixture(case["head"]), allow_pickle=False)


def detect_case(g, case):
    cfg = json.loads(str(g["cfg"]))
    head, C = cfg["head"], cfg["num_classes"]
    A = len(head["sizes"]) * len(head["rotations"])
    maps = [pp_detect_maps(s, case["H"], case["W"], C, A, head["rotations"], head["dir_offset"], case["n_fg"],
                           case["empty_classes"]) for s in case["seeds"]]
    cls, reg, dir_ = (torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3))
    return cfg, cls, reg, dir_


def reference(g, name, b):
    k = "det_%s_%d_" % (name, b)
    return g[k + "boxes"], g[k + "scores"], g[k + "labels"]


def test_detect_cases_cover_the_heads():
    for k, C, A in (("nuscenes", 7, 14), ("argoverse", 5, 10), ("lyft", 9, 18)):
        g = np.load(fixture(k), allow_pickle=False)
        assert json.loads(str(g["detect_cases"])) == [c for c in DETECT_CASES if c["head"] == k]
        cfg = json.loads(str(g["cfg"]))
        h = cfg["head"]
        assert cfg["num_classes"] == C and len(h["sizes"]) * len(h["rotations"]) == A
        full = next(c for c in DETECT_CASES if c["name"] == k + "_full")
        small = next(c for c in DETECT_CASES if c["name"] == k + "_small")
        assert full["H"] == full["W"] == CONFIGS[k]["hw"]
        assert small["H"] * small["W"] * A < h["nms_pre"]
        assert small["empty_classes"][0] not in reference(g, small["name"], 0)[2]    # nothing above score_thr
        if k != "lyft":
            assert h["dir_offset"] == pytest.approx(0.7854)


@pytest.mark.parametrize("case", DETECT_CASES, ids=[c["name"] for c in DETECT_CASES])
def test_oracle_get_bboxes_matches_reference_fixture(case):
    g = head_fixture(case)
    cfg, cls, reg, dir_ = detect_case(g, case)
    head = cfg["head"]
    anchors = grid_anchors(head, case["H"], case["W"], "cpu")
    boxes, scores, labels, m = pp_get_bboxes(cls, reg, dir_, anchors, cfg["num_classes"], head["nms_pre"],
                                             head["score_thr"], head["dir_offset"])
    assert_margins(m, topk=anchors.shape[0] > head["nms_pre"])
    for b in range(len(case["seeds"])):
        rb, rs, rl = reference(g, case["name"], b)
        assert len(rb) > 0
        assert np.array_equal(labels[b].numpy(), rl)
        np.testing.assert_allclose(scores[b].numpy(), rs, rtol=0, atol=1e-6)
        np.testing.assert_allclose(boxes[b].numpy(), rb, rtol=1e-6, atol=1e-5)
