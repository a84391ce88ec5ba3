"""The float64 rotated-box oracle (oracle/ops_ref.c: c_iou_matrix, c_nms) on the invariants the kernels are held to
in tests/test_gpu_rbox.py: closed-form IoUs at LiDAR range, translation invariance, IoU within [0, 1], and NMS at
thr = 1.0 keeping exact duplicates.  Runs without a GPU."""
import numpy as np
import pytest

from oracle import ops as O
from rbox_cases import (CLOSED_FORM_CENTRES, check_closed_forms, closed_forms, degenerate_boxes, duplicate_boxes,
                        grid_groups, paired, to_3d, translatable_boxes, vertical_cases)

ORACLE_TOL = 2e-7          # c_iou_matrix returns float32: a few ulps of values up to 1


@pytest.mark.parametrize("centre", CLOSED_FORM_CENTRES)
@pytest.mark.parametrize("mode", [0, 1])
def test_oracle_closed_forms(centre, mode):
    cases = closed_forms(*centre)
    if mode == 0:
        iou = paired(lambda a, b: O.c_iou_matrix(a, b, 0))
    else:
        iou = paired(lambda a, b: O.c_iou_matrix(to_3d(a), to_3d(b), 1))
    check_closed_forms(iou, cases, ORACLE_TOL)


def test_oracle_translation_invariance_and_range():
    a = translatable_boxes()
    m = O.c_iou_matrix(a, a, 0)
    t = a.copy()
    t[:, 0] += 64
    t[:, 1] -= 64
    assert np.array_equal(t[:, :2].astype(np.float64), a[:, :2].astype(np.float64) + [64, -64])   # exact shift
    assert np.abs(O.c_iou_matrix(t, t, 0) - m).max() <= ORACLE_TOL
    assert (m > 0).sum() > 3 * len(a)                    # the clusters overlap
    assert np.abs(np.diagonal(m) - 1).max() <= ORACLE_TOL
    assert np.abs(m - m.T).max() <= ORACLE_TOL


def test_oracle_iou_stays_in_unit_interval():
    for _, a, b in grid_groups():
        m = O.c_iou_matrix(a, b, 0)
        assert m.min() >= 0 and m.max() <= 1
        assert O.c_iou_matrix(a, a, 0).max() <= 1
    d = degenerate_boxes()
    for mode, x in ((0, d), (1, to_3d(d))):
        m = O.c_iou_matrix(x, x, mode)
        assert (m[:-1] == 0).all() and (m[:, :-1] == 0).all() and m[-1, -1] == 1


def test_oracle_iou_3d_vertical_overlap():
    for name, a, b, want in vertical_cases():
        got = O.c_iou_matrix(a[None], b[None], 1)[0, 0]
        assert abs(got - want) <= ORACLE_TOL, (name, got, want)
        assert abs(O.c_iou_matrix(b[None], a[None], 1)[0, 0] - want) <= ORACLE_TOL, name


def test_oracle_nms_keeps_exact_duplicates_at_thr_one():
    boxes, scores = duplicate_boxes()
    keep, _ = O.c_nms(boxes, scores, 1.0)
    assert keep.tolist() == list(range(len(boxes)))
    keep, _ = O.c_nms(boxes, scores, 0.99)
    assert keep.tolist() == list(range(0, len(boxes), 3))
    keep, _ = O.c_nms(boxes, scores, -0.5)
    assert keep.tolist() == [0]
