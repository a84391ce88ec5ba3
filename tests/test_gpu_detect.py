"""PointPillars box decoding on the device (detect.cu through PointPillarsB200.get_bboxes / get_bboxes_padded):
against the unmodified reference's get_bboxes (tests/golden/boundary_pointpillars_detect.npz), against the oracle
restatement detect_support.pp_get_bboxes with the same anchors, batch invariance, no host synchronisation,
CUDA-graph capture and argument errors.

Tolerances are about 5x the largest error measured on an H100 80GB HBM3; the measured value is quoted beside each.
Boxes are compared as max |got - want| / max(1, |want|) per coordinate (positions reach 75 m), scores absolutely."""
import json

import numpy as np
import pytest
import torch

from detect_support import pp_detect_maps, pp_get_bboxes
from helpers import golden, state_dict
from test_oracle_detect import CASES, assert_margins, detect_case, reference

pytestmark = pytest.mark.gpu

# largest errors measured on an H100 80GB HBM3 over every comparison below: boxes 2.4e-7, scores 1.2e-7 (1 ulp of 1.0)
BOX_TOL = 1.2e-6
SCORE_TOL = 6e-7


def box_err(got, want):
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    if want.numel() == 0:
        return 0.0
    return float(((got - want).abs() / want.abs().clamp_min(1.0)).max())


def score_err(got, want):
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    return float((got - want).abs().max()) if want.numel() else 0.0


def detector(head, num_classes, seed=1):
    """A PointPillarsB200 whose head has len(sizes) * len(rotations) anchors x num_classes classes (the KITTI
    manifest's weights, the class conv cut to the class count)."""
    import open3d_ml_b200 as M
    sd, extra = state_dict("pointpillars_kitti.manifest.json", seed)
    A = len(head["sizes"]) * len(head["rotations"])
    assert sd["bbox_head.conv_reg.weight"].shape[0] == 7 * A
    for k in ("weight", "bias"):
        sd["bbox_head.conv_cls." + k] = sd["bbox_head.conv_cls." + k][:A * num_classes].contiguous()
    return M.PointPillarsB200(sd, dict(extra["cfg"], head=head, num_classes=num_classes))


def fixture_heads():
    g = golden("boundary_pointpillars_detect.npz")
    return {k: json.loads(str(g["cfg_" + k])) for k in ("kitti", "waymo")}


# ----------------------------------------------------------------------------------- vs the reference's get_bboxes
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_fused_get_bboxes_matches_reference_fixture(case):
    g = golden("boundary_pointpillars_detect.npz")
    cfg, cls, reg, dir_ = detect_case(g, case)
    head = cfg["head"]
    net = detector(head, cfg["num_classes"])
    anchors = net.anchors(case["H"], case["W"], "cuda")
    _, _, _, m = pp_get_bboxes(cls, reg, dir_, anchors.cpu(), cfg["num_classes"], head["nms_pre"],
                                  head["score_thr"], head["dir_offset"])
    assert_margins(m, topk=anchors.shape[0] > head["nms_pre"])
    boxes, scores, labels = net.get_bboxes(cls.cuda(), reg.cuda(), dir_.cuda())
    for b in range(len(case["seeds"])):
        rb, rs, rl = reference(g, case["name"], b)
        assert len(boxes[b]) == len(rb) > 0
        assert torch.equal(labels[b].cpu(), torch.from_numpy(rl))
        be, se = box_err(boxes[b], rb), score_err(scores[b], rs)
        assert be < BOX_TOL and se < SCORE_TOL, (be, se)


# ------------------------------------------------------------------------------------------------ vs the oracle
EDGE = dict(
    kitti=dict(head="kitti", H=64, W=80, C=None, n_fg=160),
    waymo=dict(head="waymo", H=200, W=240, C=None, n_fg=4400),                     # nonzero dir_offset, K = 4096
    tie=dict(head="kitti", H=64, W=80, C=None, n_fg=200, saturate=150),           # score 1.0 across the top-k boundary
    single_class=dict(head="kitti", H=64, W=80, C=1, n_fg=160),
    one_pixel=dict(head="kitti", H=1, W=1, C=None, n_fg=4),                       # linspace with one step, N < nms_pre
    overlap=dict(head="kitti", H=2, W=2, C=None, n_fg=24, box="overlap"),         # one survivor per class
    disjoint=dict(head="waymo", H=20, W=20, C=None, n_fg=2000, box="disjoint"),   # every box above score_thr survives
    empty=dict(head="kitti", H=64, W=80, C=None, n_fg=0),
)


def edge_maps(spec, seeds, C, A, head):
    maps = [pp_detect_maps(s, spec["H"], spec["W"], C, A, head["rotations"], head["dir_offset"], spec["n_fg"],
                           saturate=spec.get("saturate", 0), box=spec.get("box", "clustered")) for s in seeds]
    return [torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3)]


def compare_with_oracle(net, cls, reg, dir_, C, head, name, exact_ties=False, topk=True):
    anchors = net.anchors(cls.shape[2], cls.shape[3], "cuda")
    wb, ws, wl, m = pp_get_bboxes(cls, reg, dir_, anchors.cpu(), C, head["nms_pre"], head["score_thr"],
                                     head["dir_offset"])
    assert_margins(m, topk=topk and anchors.shape[0] > head["nms_pre"], exact_ties=exact_ties)
    boxes, scores, labels = net.get_bboxes(cls.cuda(), reg.cuda(), dir_.cuda())
    for b in range(cls.shape[0]):
        assert len(boxes[b]) == len(wb[b])
        assert torch.equal(labels[b].cpu(), wl[b])
        be, se = box_err(boxes[b], wb[b]), score_err(scores[b], ws[b])
        assert be < BOX_TOL and se < SCORE_TOL, (b, be, se)
    return boxes, labels


# The Waymo case runs at B = 1 only: its smallest |IoU - 0.01| over 3 x 4096 boxes per frame falls below IOU_NOISE
# once several frames are pooled.
@pytest.mark.parametrize("name,B", [(n, B) for n in EDGE for B in ((1,) if n == "waymo" else (1, 3, 8))])
def test_fused_get_bboxes_matches_oracle(name, B):
    spec = EDGE[name]
    head = fixture_heads()[spec["head"]]
    C = spec["C"] or head["num_classes"]
    h = head["head"]
    A = len(h["sizes"]) * len(h["rotations"])
    net = detector(h, C)
    cls, reg, dir_ = edge_maps(spec, [1000 * B + 17 * b + len(name) for b in range(B)], C, A, h)
    boxes, labels = compare_with_oracle(net, cls, reg, dir_, C, h, name, exact_ties="saturate" in spec,
                                        topk=spec["n_fg"] > 0)     # with nothing above score_thr the top-k cut is moot
    for b in range(B):
        n_c = torch.bincount(labels[b].cpu(), minlength=C)
        if name == "empty":
            assert len(boxes[b]) == 0
        elif name == "overlap":
            assert n_c.tolist() == [1] * C
        elif name == "disjoint":
            assert int((cls[b].view(A, C, -1).sigmoid() > h["score_thr"]).sum()) == len(boxes[b])
        elif name == "tie":
            assert labels[b].numel() > 0


# --------------------------------------------------------------------------- invariance, syncs, graphs, padding
def test_batch_invariance_and_repeatability():
    head = fixture_heads()["waymo"]["head"]
    net = detector(head, 3)
    cls, reg, dir_ = (t.cuda() for t in edge_maps(EDGE["waymo"], list(range(40, 48)), 3, 6, head))
    full = net.get_bboxes_padded(cls, reg, dir_)
    again = net.get_bboxes_padded(cls, reg, dir_)
    for x, y in zip(full, again):
        assert torch.equal(x, y)
    for b in (0, 5, 7):
        one = net.get_bboxes_padded(cls[b:b + 1], reg[b:b + 1], dir_[b:b + 1])
        for x, y in zip(one, full):
            assert torch.equal(x[0], y[b])


def test_no_sync_graph_capture_and_padding():
    head = fixture_heads()["kitti"]["head"]
    net = detector(head, 3)
    maps = [t.cuda() for t in edge_maps(EDGE["kitti"], [5, 6, 7], 3, 6, head)]
    eager = net.get_bboxes_padded(*maps)              # builds the anchor cache
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = net.get_bboxes_padded(*maps)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for x, y in zip(out, eager):
        assert torch.equal(x, y)
    boxes, scores, labels, counts = eager
    for b, n in enumerate(counts.tolist()):
        assert 0 < n < labels.shape[1]
        assert bool((labels[b, n:] == -1).all()) and bool((scores[b, n:] == 0).all()) and bool((boxes[b, n:] == 0).all())
        assert bool((labels[b, :n] >= 0).all())
    static = [m.clone() for m in maps]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        net.get_bboxes_padded(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = net.get_bboxes_padded(*static)
    new = [t.cuda() for t in edge_maps(EDGE["kitti"], [8, 9, 10], 3, 6, head)]
    for dst, src in zip(static, new):
        dst.copy_(src)
    graph.replay()
    want = net.get_bboxes_padded(*new)
    torch.cuda.synchronize()
    for x, y in zip(captured, want):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------- end to end
def test_fused_forward_then_get_bboxes_matches_oracle_on_fused_maps():
    import open3d_ml_b200 as M
    from oracle import weights
    g = golden("boundary_pointpillars_class.npz")
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), int(g["weight_seed"]))
    cfg = dict(json.loads(str(g["cfg"])), **{k: fixture_heads()["kitti"][k] for k in ("head", "num_classes")})
    net = M.PointPillarsB200(sd, cfg)
    cls, reg, dir_ = net([torch.from_numpy(g["point_%d" % i]).cuda() for i in range(int(g["frames"]))])
    compare_with_oracle(net, cls.cpu(), reg.cpu(), dir_.cpu(), cfg["num_classes"], cfg["head"], "end_to_end",
                        exact_ties=True)


# ------------------------------------------------------------------------------------------------------ errors
def test_errors():
    import open3d_ml_b200 as M
    heads = fixture_heads()
    head = heads["kitti"]["head"]
    net = detector(head, 3)
    cls, reg, dir_ = (t.cuda() for t in edge_maps(EDGE["kitti"], [1], 3, 6, head))
    with pytest.raises(RuntimeError):
        net.get_bboxes_padded(cls[:, :12], reg, dir_)                   # bad channel count
    with pytest.raises(RuntimeError):
        net.get_bboxes_padded(cls, reg[:, :35], dir_)
    with pytest.raises(RuntimeError):
        detector(head, 2).get_bboxes_padded(cls, reg, dir_)             # head has 2 classes, maps 3
    sd, extra = state_dict("pointpillars_kitti.manifest.json", 1)
    bare = M.PointPillarsB200(sd, extra["cfg"])                         # the manifests' cfg: no head section
    with pytest.raises(RuntimeError, match="head"):
        bare.get_bboxes(cls, reg, dir_)
    big = detector(dict(head, nms_pre=4097), 3)
    with pytest.raises(RuntimeError, match="nms_pre"):
        big.get_bboxes_padded(cls, reg, dir_)
    ok = detector(dict(head, nms_pre=4096), 3)
    assert ok.get_bboxes_padded(cls, reg, dir_)[0].shape == (1, 3 * 4096, 7)
