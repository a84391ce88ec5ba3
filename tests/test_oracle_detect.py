"""detect_support.pp_get_bboxes against the unmodified Anchor3DHead.get_bboxes recorded in
tests/golden/boundary_pointpillars_detect.npz (`python tests/ref_detect_case.py --ops oracle --record tests/golden`):
labels and order exact, boxes and scores within fp32 rounding.  The maps are regenerated from the recorded case specs
by detect_support.pp_detect_maps.  Runs without a GPU."""
import json

import numpy as np
import pytest
import torch

from detect_support import pp_detect_maps, pp_get_bboxes
from helpers import golden
from open3d_ml_b200.pointpillars import grid_anchors

FP32_NOISE = 1e-6          # scores are in [0, 1]: a few ulps of 1.0; the yaw fraction is O(1)
IOU_NOISE = 1e-5           # IoU of metre-sized boxes from fp32 corners at |x| <= 75 m: a few 1e-6


def detect_case(g, case):
    cfg = json.loads(str(g["cfg_" + case["head"]]))
    head, C = cfg["head"], cfg["num_classes"]
    A = len(head["sizes"]) * len(head["rotations"])
    maps = [pp_detect_maps(s, case["H"], case["W"], C, A, head["rotations"], head["dir_offset"], case["n_fg"],
                           case["empty_classes"]) for s in case["seeds"]]
    cls, reg, dir_ = (torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3))
    return cfg, cls, reg, dir_


def reference(g, name, b):
    k = "%s_%d_" % (name, b)
    return g[k + "boxes"], g[k + "scores"], g[k + "labels"]


def assert_margins(m, topk=True, exact_ties=False):
    """topk: the top-k boundary decides (N > nms_pre); exact_ties: a gap of exactly 0 is an exact tie (saturated
    scores), which the (score, row) rule resolves the same way on both sides."""
    if topk and not (exact_ties and m["topk_gap"] == 0):
        assert m["topk_gap"] > FP32_NOISE, m
    assert m["thr_gap"] > FP32_NOISE and m["nms_gap"] > IOU_NOISE and m["dir_gap"] > FP32_NOISE, m


CASES = json.loads(str(golden("boundary_pointpillars_detect.npz")["cases"]))


def test_fixture_covers_the_issue_cases():
    g = golden("boundary_pointpillars_detect.npz")
    kitti, waymo = json.loads(str(g["cfg_kitti"])), json.loads(str(g["cfg_waymo"]))
    assert kitti["head"]["nms_pre"] == 100 and kitti["num_classes"] == 3
    assert waymo["head"]["nms_pre"] == 4096 and waymo["head"]["dir_offset"] == pytest.approx(0.7854)
    small = next(c for c in CASES if c["name"] == "small")
    assert small["H"] * small["W"] * 6 < waymo["head"]["nms_pre"]
    assert 1 not in reference(g, "small", 0)[2]          # a class with nothing above score_thr


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_get_bboxes_matches_reference_fixture(case):
    g = golden("boundary_pointpillars_detect.npz")
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
