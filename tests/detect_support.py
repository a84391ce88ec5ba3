"""PointPillars box decoding: test support shared by tests/test_oracle_detect.py, tests/test_gpu_detect.py,
tests/ref_detect_case.py (which records tests/golden/boundary_pointpillars_detect.npz) and bench_detect.py.

  * pp_get_bboxes: plain-torch restatement of Anchor3DHead.get_bboxes (ml3d/torch/models/point_pillars.py:945-1025,
    multiclass_nms objdet_helper.py:316-350) from the contract of DESIGN.md section 2, with its decision margins;
  * pp_detect_maps: seeded synthetic head maps whose decisions clear fp32 noise;
  * PP_DETECT_CASES: the frames of the recorded fixture.
Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
import math

import numpy as np
import torch

from oracle import ops as O


# the frames of tests/golden/boundary_pointpillars_detect.npz; the tests regenerate their maps from these specs with
# pp_detect_maps.  "head" names the yml whose model.head / classes apply.
PP_DETECT_CASES = [
    dict(name="kitti", head="kitti", H=248, W=216, seeds=[101, 102], n_fg=160, empty_classes=[]),
    dict(name="waymo", head="waymo", H=468, W=468, seeds=[207], n_fg=4600, empty_classes=[]),
    dict(name="small", head="waymo", H=6, W=5, seeds=[301], n_fg=60, empty_classes=[1]),
]


def _c_nms_tensors(bev, scores, thr):
    keep, gap = O.c_nms(bev.detach().cpu().numpy(), scores.detach().cpu().numpy(), thr)
    return torch.from_numpy(keep).to(bev.device), gap


def pp_get_bboxes(cls, reg, dir, anchors, num_classes, nms_pre, score_thr, dir_offset, nms=_c_nms_tensors,
                  with_margins=True):
    """Anchor3DHead.get_bboxes (point_pillars.py:945-1025, multiclass_nms objdet_helper.py:316-350) restated from the
    contract of DESIGN.md section 2: cls/reg/dir NCHW head maps of B frames, anchors [H*W*A, 7].
    nms(bev [n,5] (x0, y0, x1, y1, r), scores [n], thr) -> keep (or (keep, gap)) in visiting order.
    Returns (boxes, scores, labels) lists per frame and the decision margins:
      topk_gap   smallest gap between the K-th and (K+1)-th max score of a frame (inf when every row is kept),
      thr_gap    smallest |score_c - score_thr| over the kept rows and classes,
      nms_gap    smallest |IoU - 0.01| over the NMS decisions (from nms, when it reports one),
      dir_gap    smallest distance of (yaw - dir_offset) / pi + 1 from an integer over the output boxes.
    with_margins=False skips the margins (each reads a value back to the host), for timing the flow itself."""
    C = int(num_classes)
    A = reg.shape[1] // 7
    margins = dict(topk_gap=math.inf, thr_gap=math.inf, nms_gap=math.inf, dir_gap=math.inf)
    out_b, out_s, out_l = [], [], []
    for b in range(cls.shape[0]):
        sc = cls[b].permute(1, 2, 0).reshape(-1, C).sigmoid()          # row (y * W + x) * A + a, class a * C + c
        dl = reg[b].permute(1, 2, 0).reshape(-1, 7)
        dp = dir[b].permute(1, 2, 0).reshape(-1, 2)
        an = anchors
        N = sc.shape[0]
        rows = torch.arange(N, device=sc.device)
        if N > nms_pre:
            mx = sc.max(1).values
            # (score descending, row ascending): a stable sort of the rows (ascending) by descending score
            order = torch.sort(mx, descending=True, stable=True).indices
            if with_margins:
                margins["topk_gap"] = min(margins["topk_gap"], float(mx[order[nms_pre - 1]] - mx[order[nms_pre]]))
            rows = order[:nms_pre]
        sc, dl, dp, an = sc[rows], dl[rows], dp[rows], an[rows]
        dirc = (dp[:, 1] > dp[:, 0]).to(torch.float32)                  # argmax, ties -> 0
        # BBoxCoder.decode: anchors (x, y, z, w, l, h, r), deltas (dx, dy, dz, dw, dl, dh, dr)
        ha = an[:, 5]
        diag = torch.sqrt(an[:, 4] * an[:, 4] + an[:, 3] * an[:, 3])
        hg = torch.exp(dl[:, 5]) * ha
        box = torch.stack([dl[:, 0] * diag + an[:, 0], dl[:, 1] * diag + an[:, 1],
                           (dl[:, 2] * ha + (an[:, 2] + ha / 2)) - hg / 2,
                           torch.exp(dl[:, 3]) * an[:, 3], torch.exp(dl[:, 4]) * an[:, 4], hg, dl[:, 6] + an[:, 6]], 1)
        bb, ss, ll = [], [], []
        for c in range(C):
            s_c = sc[:, c]
            if with_margins and len(s_c):
                margins["thr_gap"] = min(margins["thr_gap"], float((s_c - score_thr).abs().min()))
            idx = torch.nonzero(s_c > score_thr).reshape(-1)
            if len(idx) == 0:
                continue
            x = box[idx]
            bev = torch.stack([x[:, 0] - x[:, 3] / 2, x[:, 1] - x[:, 4] / 2, x[:, 0] + x[:, 3] / 2,
                               x[:, 1] + x[:, 4] / 2, x[:, 6]], 1)
            res = nms(bev, s_c[idx], 0.01)
            if isinstance(res, tuple):
                res, gap = res
                margins["nms_gap"] = min(margins["nms_gap"], gap)
            k = idx[torch.as_tensor(res, device=idx.device).long()]
            v = box[k].clone()
            t = v[:, 6] - dir_offset
            if with_margins:
                margins["dir_gap"] = min([margins["dir_gap"]] + [abs(q - round(q)) for q in
                                                                 (t.double() / math.pi + 1).tolist()])
            v[:, 6] = (t - torch.floor(t / math.pi + 1) * math.pi) + dir_offset + math.pi * dirc[k]
            bb.append(v)
            ss.append(s_c[k])
            ll.append(torch.full((len(k),), c, dtype=torch.int64, device=v.device))
        dev = cls.device
        out_b.append(torch.cat(bb) if bb else torch.zeros((0, 7), device=dev))
        out_s.append(torch.cat(ss) if ss else torch.zeros((0,), device=dev))
        out_l.append(torch.cat(ll) if ll else torch.zeros((0,), dtype=torch.int64, device=dev))
    return out_b, out_s, out_l, margins


def pp_detect_maps(seed, H, W, C, A, rotations, dir_offset, n_fg, empty_classes=(), saturate=0, box="clustered"):
    """Seeded PointPillars head maps of ONE frame (cls [A*C, H, W], reg [A*7, H, W], dir [A*2, H, W], float32 numpy)
    whose box-decoding decisions clear fp32 noise:
      * n_fg foreground rows (clustered around a few centres) carry class logits from one shuffled grid of
        spacing 2.5e-4 in [-1.8, 5]; every other logit lies in [-9, -3.5] (scores < 0.03, far below a 0.1 threshold),
        so neither the top-k boundary nor a class's score threshold sits on a near-tie;
      * the first `saturate` foreground rows have every class logit at 30 (score exactly 1.0: exact top-k ties);
      * yaw deltas put (yaw - dir_offset) / pi at least 0.15 / pi away from an integer;
      * box "clustered": sizes within exp(+-0.2) of the anchor; "overlap": 1000x the anchor (every pair of a small map overlaps);
        "disjoint": 1/1000 of the anchor, each anchor of a pixel shifted by its own offset (no pair overlaps)."""
    rng = np.random.default_rng(seed)
    R = len(rotations)
    N = H * W * A
    cls = rng.uniform(-9.0, -3.5, (N, C)).astype(np.float32)
    n_fg = min(n_fg, N)
    if n_fg:
        centres = rng.integers(0, [H, W], (max(1, n_fg // 10), 2))
        picked, seen = [], set()
        while len(picked) < n_fg:
            cy, cx = centres[rng.integers(len(centres))]
            y = int(np.clip(cy + rng.normal(0, 3), 0, H - 1))
            x = int(np.clip(cx + rng.normal(0, 3), 0, W - 1))
            r = (y * W + x) * A + int(rng.integers(A))
            if r not in seen:
                seen.add(r)
                picked.append(r)
            elif len(seen) >= N:
                break
        picked = np.array(picked)
        grid = rng.permutation(np.arange(-1.8, 5.0, 2.5e-4))[:n_fg * C].reshape(n_fg, C)
        on = rng.random((n_fg, C)) < 0.6
        on[np.arange(n_fg), rng.integers(0, C, n_fg)] = True
        cls[picked] = np.where(on, grid, cls[picked]).astype(np.float32)
        cls[picked[:saturate]] = 30.0
    for c in empty_classes:
        cls[:, c] = rng.uniform(-9.0, -3.5, N)
    reg = rng.normal(0, 0.2, (N, 7)).astype(np.float32)
    if box == "overlap":
        reg[:, 3:5] = np.log(1000.0)
    elif box == "disjoint":
        reg[:, 3:5] = np.log(0.001)
        reg[:, 0] = (np.arange(N) % A) * 0.2
        reg[:, 1] = 0
    rot_a = np.tile(np.asarray(rotations, np.float64), A // R)[np.arange(N) % A]
    v = rng.uniform(0.15, np.pi - 0.15, N) - np.pi * rng.integers(0, 2, N)
    reg[:, 6] = (v + dir_offset - rot_a).astype(np.float32)
    d = rng.normal(0, 1, (N, 2)).astype(np.float32)

    def nchw(a):       # rows (y * W + x) * A + a, channel a * k + j  ->  [A * k, H, W]
        return np.ascontiguousarray(a.reshape(H, W, -1).transpose(2, 0, 1))
    return nchw(cls), nchw(reg), nchw(d)
