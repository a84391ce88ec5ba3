"""Rotated-box IoU and NMS cases shared by tests/test_gpu_rbox.py (the kernels of rbox.cuh / nms.cu / detect.cu) and
tests/test_oracle_rbox.py (the float64 oracle, oracle/ops_ref.c).  Boxes are float32 numpy arrays:
  * (x, y, w, h, r) rows for iou_bev, (x, y, z, w, h, l, ry) rows for iou_3d,
  * (x0, y0, x1, y1, r) rows for nms.
Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
import math

import numpy as np

from oracle import ops as O

# Absolute IoU tolerances of the kernel-vs-oracle comparisons, about 5x the largest |IoU_fp32 - IoU_f64| measured on an
# H100 80GB HBM3 (700 W power limit) over tests/test_gpu_rbox.py.  The error grows with the aspect ratio (a heading
# rounded to fp32 turns a long thin box by ~1e-7 rad, which moves its overlap in proportion to length / width):
#   boxes of aspect <= 10 (every detection box): measured 6.6e-7 (3.6e-7 at aspect 1), closed forms 1.5e-7;
#   aspect 100: measured 5.7e-6.
IOU_TOL = 3.5e-6
IOU_TOL_ASPECT100 = 3e-5

CENTRES = (0.0, 8.0, 40.0, 75.0, 150.0)
QUADRANTS = ((1, 1), (-1, 1), (-1, -1), (1, -1))
SIZES = (0.05, 0.1, 0.6, 4.0, 20.0)
ASPECTS = (1, 10, 100)
FAR_HEADINGS = (3 * math.pi, -3 * math.pi, 50.0, -50.0)     # sincosf's full range reduction
CLOSED_FORM_CENTRES = ((0.0, 0.0), (70.1, -39.6))


def to_3d(bev, y=0.5, h=1.0):
    """(x, y, w, h, r) -> (x, y, z, w, h, l, ry) with the footprint in the ground plane (x, z) and every box spanning
    the same height [y - h, y]: the 3-D IoU is then the BEV IoU."""
    bev = np.asarray(bev, np.float32)
    n = len(bev)
    return np.stack([bev[:, 0], np.full(n, y), bev[:, 1], bev[:, 2], np.full(n, h), bev[:, 3], bev[:, 4]],
                    1).astype(np.float32)


def to_xyxyr(bev):
    bev = np.asarray(bev, np.float64)
    return np.stack([bev[:, 0] - bev[:, 2] / 2, bev[:, 1] - bev[:, 3] / 2, bev[:, 0] + bev[:, 2] / 2,
                     bev[:, 1] + bev[:, 3] / 2, bev[:, 4]], 1).astype(np.float32)


# ------------------------------------------------------------------------------------------------------ IoU grid
def grid_group(centre, quadrant, size, aspect, n=24, seed=0):
    """Two sets of n boxes whose centres lie within one box size of (qx * centre, qy * centre): short side about
    `size`, long side about `size * aspect`, headings uniform in [-pi, pi] with FAR_HEADINGS mixed in.  Most pairs
    overlap."""
    rng = np.random.default_rng(seed)
    c = np.array([quadrant[0] * centre, quadrant[1] * centre])

    def one():
        w = size * rng.uniform(0.7, 1.3, n)
        h = w * aspect * rng.uniform(0.8, 1.25, n)
        swap = rng.random(n) < 0.5
        w, h = np.where(swap, h, w), np.where(swap, w, h)
        xy = c + rng.uniform(-size, size, (n, 2))
        r = rng.uniform(-math.pi, math.pi, n)
        r[rng.choice(n, len(FAR_HEADINGS), replace=False)] = FAR_HEADINGS
        return np.concatenate([xy, w[:, None], h[:, None], r[:, None]], 1).astype(np.float32)
    return one(), one()


def grid_tol(name):
    """The tolerance of a grid group by the aspect ratio in its name."""
    return IOU_TOL_ASPECT100 if name.endswith(" a100") else IOU_TOL


def grid_groups():
    """(name, a, b) over the range x size x aspect grid."""
    seed = 0
    for centre in CENTRES:
        for quadrant in (QUADRANTS[:1] if centre == 0 else QUADRANTS):
            for size in SIZES:
                for aspect in ASPECTS:
                    seed += 1
                    a, b = grid_group(centre, quadrant, size, aspect, seed=seed)
                    yield "c%g q%d%d s%g a%d" % (centre, quadrant[0], quadrant[1], size, aspect), a, b


# ------------------------------------------------------------------------------------------------- closed forms
def closed_forms(cx, cy):
    """(name, a [5], b [5], kind, value) in the (x, y, w, h, r) form around the float32 centre (cx, cy).
    kind "eq": IoU == value; "le": IoU <= value (touching boxes: a degenerate intersection); "zero": IoU == 0 exactly.
    Sizes and axis-aligned offsets are short dyadic numbers, so that the shifted float32 centres are exact."""
    c = np.float32([cx, cy]).astype(np.float64)
    w, h = 0.625, 0.75                           # about a KITTI pedestrian (0.6 x 0.8)
    r = 0.3
    r32 = float(np.float32(r))
    half_pi = float(np.float32(math.pi / 2))     # cos(float(pi/2)) = -4.4e-8: offsets along its axes stay exact enough
    quarter_pi = float(np.float32(math.pi / 4))
    oct_area = 2 * (math.sqrt(2) - 1) * 4.0      # a 2 x 2 square and itself turned by 45 degrees: the regular octagon

    def box(dx, dy, bw, bh, br):
        return np.float32([c[0] + dx, c[1] + dy, bw, bh, br])
    cases = [
        ("identical", box(0, 0, w, h, r), box(0, 0, w, h, r), "eq", 1.0),
        ("identical_axis", box(0, 0, 4, 1.5, 0), box(0, 0, 4, 1.5, 0), "eq", 1.0),
        ("swapped_wh", box(0, 0, w, h, r), box(0, 0, h, w, r32 + math.pi / 2), "eq", 1.0),
        ("r_plus_pi", box(0, 0, w, h, r), box(0, 0, w, h, r32 + math.pi), "eq", 1.0),
        ("nested_concentric", box(0, 0, 4, 1.5, r), box(0, 0, 1, 0.5, r), "eq", 0.5 / 6),
        ("nested_offset", box(0, 0, 4, 1.5, 0), box(1, 0.25, 1, 0.5, 0), "eq", 0.5 / 6),
        ("half_overlap_x", box(0, 0, w, h, 0), box(w / 2, 0, w, h, 0), "eq", 1 / 3),
        ("half_overlap_y", box(0, 0, w, h, half_pi), box(0, w / 2, w, h, half_pi), "eq", 1 / 3),
        ("octagon", box(0, 0, 2, 2, 0), box(0, 0, 2, 2, quarter_pi), "eq", oct_area / (8 - oct_area)),
        ("shared_edge", box(0, 0, w, h, 0), box(w, 0, w, h, 0), "le", 0.0),
        ("shared_edge_rotated", box(0, 0, w, h, half_pi), box(0, w, w, h, half_pi), "le", 0.0),
        ("shared_corner", box(0, 0, w, h, 0), box(w, h, w, h, 0), "le", 0.0),
        ("separated_x", box(0, 0, w, h, 0), box(w + 1e-3, 0, w, h, 0), "zero", 0.0),
        ("separated_y", box(0, 0, w, h, 0), box(0, h + 1e-3, w, h, 0), "zero", 0.0),
        ("separated_rotated", box(0, 0, w, h, r),
         box((w + 1e-3) * math.cos(r32), (w + 1e-3) * math.sin(r32), w, h, r), "zero", 0.0),
        ("rotated_1e-7", box(0, 0, w, h, 0), box(0, 0, w, h, 1e-7), "eq", 1.0),    # nearly collinear edges
    ]
    return cases


def closed_form_errors(iou, cases):
    """iou(a [n,5], b [n,5]) -> [n] paired IoUs.  Returns (name, got, want, kind) for every case."""
    a = np.stack([x[1] for x in cases])
    b = np.stack([x[2] for x in cases])
    got = iou(a, b)
    return [(name, float(g), float(v), kind) for (name, _, _, kind, v), g in zip(cases, got)]


def check_closed_forms(iou, cases, tol):
    for name, got, want, kind in closed_form_errors(iou, cases):
        if kind == "eq":
            assert abs(got - want) <= tol, (name, got, want)
        elif kind == "le":
            assert 0.0 <= got <= tol, (name, got)
        else:
            assert got == 0.0, (name, got)


def paired(iou_matrix):
    """Wraps an all-pairs iou(a, b) -> [n, m] as a paired one (the diagonal)."""
    return lambda a, b: np.diagonal(iou_matrix(a, b)).copy()


# ---------------------------------------------------------------------------------------------------- invariants
def translatable_boxes(n=96, seed=5):
    """Boxes whose centres and sizes are multiples of 2^-16 with |x|, |y| < 100: shifted by (64, -64) they stay exact
    in float32.  Clusters at several ranges, sizes from 5 cm to 4 m, overlapping partners."""
    rng = np.random.default_rng(seed)
    q = 2.0 ** -16
    out = []
    for cx, cy in ((0, 0), (3, -2), (-20, 35), (36, -30)):
        for size in (0.05, 0.1, 0.6, 4.0):
            k = n // 16
            xy = np.array([cx, cy]) + rng.uniform(-size, size, (k, 2))
            wh = size * rng.uniform(0.6, 1.6, (k, 2))
            r = rng.uniform(-math.pi, math.pi, (k, 1))
            out.append(np.concatenate([np.round(xy / q) * q, np.round(wh / q) * q, r], 1))
    return np.concatenate(out).astype(np.float32)


def degenerate_boxes():
    """Boxes with a zero or negative side, and a regular partner at the same centre."""
    return np.float32([[1, 1, 0, 2, 0.2], [1, 1, 2, 0, 0.2], [1, 1, -1, 2, 0.2], [1, 1, 2, -1, 0.2], [1, 1, 0, 0, 0],
                       [1, 1, -2, -2, 0.5], [1, 1, 2, 2, 0.2]])


def vertical_cases():
    """(name, a [7], b [7], value) for iou_3d: the same 2 x 1 footprint, (x, y, z, w, h, l, ry) with the box spanning
    [y - h, y]."""
    def box(y, h):
        return np.float32([70.5, y, -39.5, 2, h, 1, 0.4])
    return [
        ("touching", box(1, 1), box(2, 1), 0.0),
        ("nested_heights", box(2, 2), box(1.25, 0.5), 0.25),
        ("half_height", box(2, 2), box(1, 2), 1 / 3),
        ("zero_height", box(1, 1), box(1, 0), 0.0),
        ("zero_height_both", box(1, 0), box(1, 0), 0.0),
    ]


# ----------------------------------------------------------------------------------------------------------- nms
def signed_gap(a, b, thr):
    """Oracle IoU(a, b) - thr for two (x0, y0, x1, y1, r) boxes (from c_nms's reported gap and decision)."""
    keep, gap = O.c_nms(np.stack([a, b]), np.float32([1.0, 0.5]), thr)
    return gap if len(keep) == 1 else -gap


def place_by_bisection(a, make_b, thr, target, t_hi=4.0):
    """Returns the float32 box make_b(t) whose oracle IoU with a is thr + target, t in [0, t_hi] found by bisection
    (the overlap of two convex boxes falls monotonically as one moves away from the other's centre)."""
    lo, hi = 0.0, t_hi
    assert signed_gap(a, make_b(lo), thr) > target > signed_gap(a, make_b(hi), thr)
    for _ in range(60):
        mid = 0.5 * (lo + hi)
        if signed_gap(a, make_b(mid), thr) > target:
            lo = mid
        else:
            hi = mid
    return make_b(hi)


def near_threshold_pairs(thr, deltas=(1e-4, 3e-4, 1e-3), reps=4, seed=0, x=69.0, w=0.6, h=0.8):
    """Pairs of pedestrian-sized boxes at x ~ 69 m, one pair every 2.5 m in y, whose float64 IoU is thr +- delta.
    Returns (boxes [2P, 5] in the (x0, y0, x1, y1, r) form, scores [2P], signed gaps [P]); the first box of a pair has
    the higher score."""
    rng = np.random.default_rng(seed)
    boxes, gaps = [], []
    k = 0
    for d in deltas:
        for sign in (1, -1):
            for _ in range(reps):
                cx, cy = x + rng.uniform(0, 0.5), -30 + 2.5 * k
                ra = rng.uniform(-math.pi, math.pi)
                # at thr = 0.5 the partner needs a near-parallel heading to reach IoU 0.5 at all
                rb = ra + (rng.uniform(-0.2, 0.2) if thr > 0.1 else rng.uniform(-math.pi, math.pi))
                phi = rng.uniform(-math.pi, math.pi)
                s = rng.uniform(0.95, 1.05)
                a = to_xyxyr([[cx, cy, w, h, ra]])[0]

                def make_b(t):
                    return to_xyxyr([[cx + t * math.cos(phi), cy + t * math.sin(phi), w * s, h * s, rb]])[0]
                b = place_by_bisection(a, make_b, thr, sign * d)
                boxes += [a, b]
                gaps.append(signed_gap(a, b, thr))
                k += 1
    P = len(gaps)
    scores = (1.0 - np.arange(2 * P) / (4.0 * P)).astype(np.float32)
    return np.stack(boxes).astype(np.float32), scores, np.array(gaps)


def chain_clusters(n, seed, step=0.3):
    """n boxes in chains of 8 (the last chain shorter): each chain shares size and heading, and box i + 1 sits
    `step * w` further along the heading than box i, so that IoUs within a chain are (w - d) / (w + d) for d = k * step * w:
    0.54, 0.25, 0.053, then 0.  Chains sit on a 6 m grid from (-60, -60).  Scores are random with exact ties, so the
    visiting order scatters every chain over several 64-box blocks."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        k, j = divmod(i, 8)
        if j == 0:
            base = np.array([-60 + 6.0 * (k % 20), -60 + 6.0 * (k // 20)]) + rng.uniform(0, 0.5, 2)
            w, h = rng.uniform(0.5, 0.6), rng.uniform(0.5, 2.0)
            r = rng.uniform(-math.pi, math.pi)
        d = j * step * w
        rows.append([base[0] + d * math.cos(r), base[1] + d * math.sin(r), w, h, r])
    boxes = to_xyxyr(rows)
    scores = rng.random(n).astype(np.float32)
    scores[n // 2:] = scores[:n - n // 2]
    perm = rng.permutation(n)
    return boxes[perm], scores


def duplicate_boxes():
    """Three exact copies of each of a few boxes, at the origin and at (70.1, -39.6), with distinct scores."""
    base = to_xyxyr([[0, 0, 0.6, 0.8, 0.3], [0, 0, 4, 1.6, -1.2], [70.1, -39.6, 0.6, 0.8, 0.3],
                     [70.1, -39.6, 4, 1.6, 2.0], [70.1, -39.6, 0.05, 5, 0.7]])
    boxes = np.repeat(base, 3, 0)
    scores = np.linspace(1, 0.1, len(boxes)).astype(np.float32)
    return boxes, scores


def limit_pairs(n_pairs=32768, seed=0):
    """2 * n_pairs boxes: n_pairs well-separated 1 x 1 boxes (3 m grid), each present twice, with distinct scores
    k / 2^16.  Returns (boxes, scores, the expected keep: the higher-scored copy of every pair by descending score)."""
    rng = np.random.default_rng(seed)
    k = np.arange(n_pairs)
    xy = np.stack([-300 + 3.0 * (k % 256), -200 + 3.0 * (k // 256)], 1)
    base = to_xyxyr(np.concatenate([xy, np.ones((n_pairs, 2)), rng.uniform(-math.pi, math.pi, (n_pairs, 1))], 1))
    idx = rng.permutation(2 * n_pairs)                 # idx[2p], idx[2p + 1]: the two copies of pair p
    boxes = np.empty((2 * n_pairs, 5), np.float32)
    boxes[idx[0::2]] = base
    boxes[idx[1::2]] = base
    scores = (rng.permutation(2 * n_pairs) / 2.0 ** 16).astype(np.float32)
    hi = np.where(scores[idx[0::2]] > scores[idx[1::2]], idx[0::2], idx[1::2])
    want = hi[np.argsort(-scores[hi], kind="stable")]
    return boxes, scores, want
