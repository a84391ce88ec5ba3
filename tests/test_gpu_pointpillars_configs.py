"""PointPillarsB200 at the nuScenes and Argoverse configs (two-layer PillarFeatureNet) and the Lyft config against
the UNMODIFIED reference class recorded in tests/golden/pointpillars_config_<k>.npz: the fused forward against the
sampled reference head maps, graphed against eager, and the fused box decoding against the reference get_bboxes on
seeded head maps of each config's head, eager and captured into a CUDA graph; and the PFN stacks the fused path
refuses."""
import pytest
import torch

from pp_configs_support import CONFIGS, DETECT_CASES, load
from test_gpu_detect import BOX_TOL, SCORE_TOL, box_err, score_err
from test_gpu_reference_boundary import TOL, sampled_rel_err
from test_oracle_pointpillars_configs import assert_margins, detect_case, head_fixture, reference

pytestmark = pytest.mark.gpu


def fused(k, **kw):
    import open3d_ml_b200 as M
    g, sd, cfg, frames = load(k)
    return M.PointPillarsB200(sd, cfg, **kw), g, [f.cuda() for f in frames]


@pytest.mark.parametrize("k", list(CONFIGS))
def test_fused_forward_matches_reference_class(k):
    net, g, frames = fused(k)
    assert net.pfn_layers == (2 if k in ("nuscenes", "argoverse") else 1)
    got = net(frames)
    errs = [sampled_rel_err(t, g, "ref_%d" % i) for i, t in enumerate(got)]
    assert all(e < TOL for e in errs), errs
    eager, _, _ = fused(k, use_graph=False)
    for a, b in zip(got, eager(frames)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("case", DETECT_CASES, ids=[c["name"] for c in DETECT_CASES])
def test_fused_get_bboxes_matches_reference(case):
    from detect_support import pp_get_bboxes
    g = head_fixture(case)
    cfg, cls, reg, dir_ = detect_case(g, case)
    head = cfg["head"]
    net, _, _ = fused(case["head"])
    anchors = net.anchors(case["H"], case["W"], "cuda")
    _, _, _, m = pp_get_bboxes(cls, reg, dir_, anchors.cpu(), cfg["num_classes"], head["nms_pre"], head["score_thr"],
                               head["dir_offset"])
    assert_margins(m, topk=anchors.shape[0] > head["nms_pre"])
    maps = [t.cuda() for t in (cls, reg, dir_)]
    boxes, scores, labels, counts = net.get_bboxes_padded(*maps)
    for b in range(len(case["seeds"])):
        rb, rs, rl = reference(g, case["name"], b)
        n = int(counts[b])
        assert n == len(rb) > 0
        assert torch.equal(labels[b, :n].cpu(), torch.from_numpy(rl))
        be, se = box_err(boxes[b, :n], rb), score_err(scores[b, :n], rs)
        assert be < BOX_TOL and se < SCORE_TOL, (be, se)
    # the same call captured into a CUDA graph and replayed
    static = [t.clone() for t in maps]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        net.get_bboxes_padded(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = net.get_bboxes_padded(*static)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(captured, (boxes, scores, labels, counts)):
        assert torch.equal(x, y)


def test_other_pfn_stacks_are_refused():
    import open3d_ml_b200 as M
    _, sd, cfg, _ = load("nuscenes")
    three = dict(sd)
    for key in [k for k in sd if k.startswith("voxel_encoder.pfn_layers.1.")]:
        three[key.replace("pfn_layers.1.", "pfn_layers.2.")] = sd[key]
    with pytest.raises(RuntimeError, match=r"\[\[32, 9\], \[64, 64\], \[64, 64\]\]"):
        M.PointPillarsB200(three, cfg)
    wide = dict(sd)
    wide["voxel_encoder.pfn_layers.1.linear.weight"] = torch.zeros(128, 64)
    with pytest.raises(RuntimeError, match=r"\[\[32, 9\], \[128, 64\]\]"):
        M.PointPillarsB200(wide, cfg)
    _, lyft, lcfg, _ = load("lyft")
    two64 = dict(lyft)                    # a [64, C+5] first layer followed by a second one
    for key in [k for k in lyft if k.startswith("voxel_encoder.pfn_layers.0.")]:
        two64[key.replace("pfn_layers.0.", "pfn_layers.1.")] = lyft[key]
    two64["voxel_encoder.pfn_layers.1.linear.weight"] = torch.zeros(64, 64)
    with pytest.raises(RuntimeError, match="not fused"):
        M.PointPillarsB200(two64, lcfg)
