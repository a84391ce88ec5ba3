"""Rotated IoU and NMS on the device (rbox.cuh through o3dml_iou_matrix, o3dml_nms and the fused PointPillars NMS of
detect.cu) against the float64 oracle (oracle/ops_ref.c) at LiDAR ranges and box edges: centres out to 150 m, boxes
from 5 cm to 20 m with aspect ratios up to 100, far headings, closed-form overlaps, touching and separated boxes,
translation and symmetry, NMS decisions within 1e-4 of the threshold, signed-zero and equal scores, and NMS at its
65 536-box limit.  The tolerances are rbox_cases.IOU_TOL and, for aspect ratio 100, IOU_TOL_ASPECT100."""
import math

import numpy as np
import pytest
import torch

from oracle import ops as O
from rbox_cases import (CLOSED_FORM_CENTRES, IOU_TOL, chain_clusters, check_closed_forms, closed_forms,
                        degenerate_boxes, duplicate_boxes, grid_groups, grid_tol, limit_pairs, near_threshold_pairs, paired,
                        signed_gap, to_3d, to_xyxyr, translatable_boxes, vertical_cases)

pytestmark = pytest.mark.gpu


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def iou_dev(a, b, mode):
    """o3dml_iou_matrix in mode 0 ([.,5] bev) or 1 ([.,7] 3d) on the device, as float32 numpy."""
    import open3d_ml_b200 as M
    got = (M.iou_bev if mode == 0 else M.iou_3d)(T(a), T(b))
    assert got.is_cuda
    return got.cpu().numpy()


def iou_pair_errors(a, b):
    """max |IoU_kernel - IoU_oracle| over a x b in both modes (mode 1 with equal height spans: the same ratio);
    every kernel IoU must lie in [0, 1]."""
    errs = []
    for mode, (x, y) in ((0, (a, b)), (1, (to_3d(a), to_3d(b)))):
        got, want = iou_dev(x, y, mode), O.c_iou_matrix(x, y, mode)
        assert got.min() >= 0 and got.max() <= 1, (mode, got.min(), got.max())
        errs.append(float(np.abs(got.astype(np.float64) - want).max()))
    return errs


# --------------------------------------------------------------------------------------------------------- IoU
@pytest.mark.parametrize("centre", [0.0, 8.0, 40.0, 75.0, 150.0])
def test_iou_range_size_grid_vs_oracle(centre):
    """Centres at `centre` m in all four quadrants x sizes 0.05 .. 20 m x aspect 1, 10, 100, headings in [-pi, pi]
    and +-3 pi, +-50 rad, partners within one box size."""
    worst = {}
    for name, a, b in grid_groups():
        if not name.startswith("c%g " % centre):
            continue
        assert (iou_dev(a, b, 0) > 0).mean() > 0.3, name          # most pairs overlap
        worst[name] = max(iou_pair_errors(a, b)) / grid_tol(name)
    assert len(worst) == (15 if centre == 0 else 60)
    name = max(worst, key=worst.get)
    assert worst[name] <= 1, (name, worst[name] * grid_tol(name))


@pytest.mark.parametrize("centre", CLOSED_FORM_CENTRES)
@pytest.mark.parametrize("mode", [0, 1])
def test_iou_closed_forms(centre, mode):
    """Identical, swapped (w, h) with r + pi/2, r and r + pi, nested, half overlap, the 45-degree octagon (8 vertices),
    shared edges and corners, 1 mm gaps (exactly 0) and a 1e-7 rad turn, at the origin and at (70.1, -39.6)."""
    cases = closed_forms(*centre)
    if mode == 0:
        iou = paired(lambda a, b: iou_dev(a, b, 0))
    else:
        iou = paired(lambda a, b: iou_dev(to_3d(a), to_3d(b), 1))
    check_closed_forms(iou, cases, IOU_TOL)
    a, b = np.stack([c[1] for c in cases]), np.stack([c[2] for c in cases])
    assert max(iou_pair_errors(a, b)) <= IOU_TOL


def test_iou_translation_symmetry_and_degenerate_boxes():
    a = translatable_boxes()
    t = a.copy()
    t[:, 0] += 64
    t[:, 1] -= 64
    assert np.array_equal(t[:, :2].astype(np.float64), a[:, :2].astype(np.float64) + [64, -64])   # exact shift
    m = iou_dev(a, a, 0)
    assert (m > 0).sum() > 3 * len(a)
    assert np.abs(iou_dev(t, t, 0) - m).max() <= IOU_TOL
    assert np.abs(m - m.T).max() <= IOU_TOL
    assert np.abs(np.diagonal(m) - 1).max() <= IOU_TOL
    for name, p, q in list(grid_groups())[::7]:
        assert np.abs(iou_dev(p, q, 0) - iou_dev(q, p, 0).T).max() <= grid_tol(name), name
    d = degenerate_boxes()
    for mode, x in ((0, d), (1, to_3d(d))):
        m = iou_dev(x, x, mode)
        assert (m[:-1] == 0).all() and (m[:, :-1] == 0).all() and abs(m[-1, -1] - 1) <= IOU_TOL


def test_iou_3d_vertical_overlap():
    for name, a, b, want in vertical_cases():
        for x, y in ((a, b), (b, a)):
            got = iou_dev(x[None], y[None], 1)[0, 0]
            assert abs(got - want) <= IOU_TOL, (name, got, want)
            if want == 0:
                assert got == 0, (name, got)


# --------------------------------------------------------------------------------------------------------- NMS
def nms_both(boxes, scores, thr):
    """The nms op on device tensors and through the CPU-tensor route; both must agree."""
    import open3d_ml_b200 as M
    got = M.nms(T(boxes), T(scores), thr)
    assert got.dtype == torch.int64 and got.is_cuda
    got_cpu = M.nms(torch.from_numpy(boxes), torch.from_numpy(scores), thr)
    assert not got_cpu.is_cuda
    assert torch.equal(got.cpu(), got_cpu)
    return got_cpu.numpy()


@pytest.mark.parametrize("n", [63, 64, 65, 127, 128, 129, 4097])
@pytest.mark.parametrize("thr", [0.01, 0.5])
def test_nms_block_edges_vs_oracle(n, thr):
    """Chains of overlapping boxes whose members scatter over several 64-box blocks of the visiting order."""
    boxes, scores = chain_clusters(n, seed=n)
    ref, gap = O.c_nms(boxes, scores, thr)
    assert gap > 5 * IOU_TOL
    assert len(ref) < n                                            # something was suppressed
    assert np.array_equal(nms_both(boxes, scores, thr), ref)


@pytest.mark.parametrize("thr", [0.01, 0.5])
def test_nms_near_threshold_pedestrians_at_range(thr):
    """Pedestrian-sized pairs at x ~ 69 m whose float64 IoU is thr +- {1e-4, 3e-4, 1e-3}: every pair's decision
    is fixed by the oracle, and half of the pairs lose their second box."""
    boxes, scores, gaps = near_threshold_pairs(thr, seed=int(thr * 100))
    assert (np.abs(gaps) > 5 * IOU_TOL).all() and (np.abs(gaps) < 2e-3).all()
    ref, gap = O.c_nms(boxes, scores, thr)
    assert gap > 5 * IOU_TOL
    assert len(ref) == len(boxes) - (gaps > 0).sum()
    assert np.array_equal(nms_both(boxes, scores, thr), ref)


def test_nms_signed_zero_and_equal_scores():
    b = to_xyxyr([[70.1, -39.6, 0.6, 0.8, 0.3]])[0]
    boxes = np.stack([b, b]).astype(np.float32)
    for scores, want in (([-0.0, 0.0], [0]), ([0.0, -0.0], [0])):
        scores = np.float32(scores)
        assert np.array_equal(O.c_nms(boxes, scores, 0.5)[0], want)
        assert np.array_equal(nms_both(boxes, scores, 0.5), want)
    # disjoint boxes: the visiting order itself is the result; +-0.0 interleaved with equal scores and a negative one
    far = to_xyxyr([[3.0 * k, 0, 1, 1, 0.1 * k] for k in range(6)])
    scores = np.float32([0.0, -0.0, -0.5, -0.0, 0.0, 0.25])
    ref, _ = O.c_nms(far, scores, 0.5)
    assert ref.tolist() == [5, 0, 1, 3, 4, 2]
    assert np.array_equal(nms_both(far, scores, 0.5), ref)
    boxes, _ = chain_clusters(300, seed=3)
    scores = np.full(300, 0.25, np.float32)
    ref, gap = O.c_nms(boxes, scores, 0.3)
    assert gap > 5 * IOU_TOL and len(ref) < 300
    assert np.array_equal(nms_both(boxes, scores, 0.3), ref)


def test_nms_duplicates_at_thr_one_and_negative_threshold():
    boxes, scores = duplicate_boxes()
    assert np.array_equal(nms_both(boxes, scores, 1.0), np.arange(len(boxes)))
    assert np.array_equal(O.c_nms(boxes, scores, 1.0)[0], np.arange(len(boxes)))
    assert np.array_equal(nms_both(boxes, scores, 0.99), np.arange(0, len(boxes), 3))
    chain, cs = chain_clusters(200, seed=4)
    for bx, sc in ((boxes, scores), (chain, cs)):
        want = [int(np.argmax(sc))]
        assert O.c_nms(bx, sc, -0.01)[0].tolist() == want
        assert nms_both(bx, sc, -0.01).tolist() == want


def test_nms_at_its_limit():
    """65 536 boxes: 32 768 well-separated pairs of duplicates, distinct scores: at thr 0.5 exactly the higher-scored
    copy of each pair survives, by descending score.  65 537 boxes are refused."""
    import open3d_ml_b200 as M
    boxes, scores, want = limit_pairs()
    got = M.nms(T(boxes), T(scores), 0.5)
    assert np.array_equal(got.cpu().numpy(), want)
    del got
    torch.cuda.empty_cache()
    more = np.concatenate([boxes, boxes[:1]])
    with pytest.raises(RuntimeError, match="65 536"):
        M.nms(T(more), T(np.concatenate([scores, scores[:1]])), 0.5)


# ---------------------------------------------------------------------------------------------- fused detection
def ped_pair_maps(seed, head, H=8, W=2, C=3):
    """One KITTI head map (cls, reg, dir as [A*C|A*7|A*2, H, W] float32) whose only boxes above score_thr are
    pedestrian-class pairs in the right-most anchor column: per pixel row, anchor 0 (rotation 0) decodes to a
    0.6 x 0.8 box at x ~ 69.9 m and anchor 1 (rotation 1.57) to a partner placed, by inverting BBoxCoder.decode and
    bisecting on the oracle, at float64 IoU 0.01 + {+2e-4, -2e-4, +1e-3, -1e-3}.  Returns the maps and the signed
    gaps."""
    from open3d_ml_b200.pointpillars import grid_anchors
    rng = np.random.default_rng(seed)
    A = len(head["sizes"]) * len(head["rotations"])
    N = H * W * A
    an = grid_anchors(head, H, W, "cpu")
    cls = rng.uniform(-9.0, -3.5, (N, C)).astype(np.float32)
    reg = np.zeros((N, 7), np.float32)
    v = rng.uniform(0.15, np.pi - 0.15, N) - np.pi * rng.integers(0, 2, N)
    reg[:, 6] = (v - an[:, 6].double().numpy()).astype(np.float32)

    def bev(row, d):
        """pp_get_bboxes' decode of one row with reg deltas d, as its (x0, y0, x1, y1, r) NMS box."""
        a, dl = an[row:row + 1], torch.from_numpy(np.float32(d)[None])
        diag = torch.sqrt(a[:, 4] * a[:, 4] + a[:, 3] * a[:, 3])
        x, y = dl[:, 0] * diag + a[:, 0], dl[:, 1] * diag + a[:, 1]
        w, l, r = torch.exp(dl[:, 3]) * a[:, 3], torch.exp(dl[:, 4]) * a[:, 4], dl[:, 6] + a[:, 6]
        return torch.stack([x - w / 2, y - l / 2, x + w / 2, y + l / 2, r], 1)[0].numpy()

    targets = (2e-4, -2e-4, 1e-3, -1e-3)
    gaps = []
    for y in range(H):
        r1, r2 = (y * W + W - 1) * A + 0, (y * W + W - 1) * A + 1
        a0 = an[r1].double().numpy()
        reg[r1, 0] = (69.9 + rng.uniform(-0.2, 0.2) - a0[0]) / 1.0          # pedestrian anchor diagonal: 1.0
        reg[r1, 1] = rng.uniform(-0.5, 0.5)
        b1 = bev(r1, reg[r1])
        cx, cy, phi = 0.5 * (b1[0] + b1[2]), 0.5 * (b1[1] + b1[3]), rng.uniform(-math.pi, math.pi)
        a1 = an[r2].double().numpy()
        diag = math.sqrt(a1[3] ** 2 + a1[4] ** 2)

        def make(t, d=reg[r2].copy()):
            d[0] = (cx + t * math.cos(phi) - a1[0]) / diag
            d[1] = (cy + t * math.sin(phi) - a1[1]) / diag
            return d
        target = targets[(y + seed) % len(targets)]
        lo, hi = 0.0, 2.0
        assert signed_gap(b1, bev(r2, make(lo)), 0.01) > target > signed_gap(b1, bev(r2, make(hi)), 0.01)
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            if signed_gap(b1, bev(r2, make(mid)), 0.01) > target:
                lo = mid
            else:
                hi = mid
        reg[r2] = make(hi)
        gaps.append(signed_gap(b1, bev(r2, reg[r2]), 0.01))
        cls[r1, 0] = 3.0 - 0.1 * y                       # distinct pedestrian scores, the first box of a pair higher
        cls[r2, 0] = 2.95 - 0.1 * y
    d = rng.normal(0, 1, (N, 2)).astype(np.float32)

    def nchw(x):
        return np.ascontiguousarray(x.reshape(H, W, -1).transpose(2, 0, 1))
    return nchw(cls), nchw(reg), nchw(d), np.array(gaps)


@pytest.mark.parametrize("B", [1, 3])
def test_fused_nms_near_threshold_pedestrians_at_range(B):
    from test_gpu_detect import compare_with_oracle, detector, fixture_heads
    cfg = fixture_heads()["kitti"]
    head, C = cfg["head"], cfg["num_classes"]
    maps = [ped_pair_maps(11 + b, head, C=C) for b in range(B)]
    for m in maps:
        gaps = m[3]
        assert (np.abs(gaps) > 1e-4).all() and (np.abs(gaps) < 2e-3).all() and (gaps > 0).any() and (gaps < 0).any()
    cls, reg, dir_ = (torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3))
    net = detector(head, C)
    boxes, labels = compare_with_oracle(net, cls, reg, dir_, C, head, "near_threshold", topk=False)
    for b, m in enumerate(maps):
        assert (labels[b] == 0).all()
        assert len(boxes[b]) == 2 * len(m[3]) - int((m[3] > 0).sum())
        assert float(boxes[b][:, 0].min()) > 68.5
