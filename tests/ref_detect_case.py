"""Records tests/golden/boundary_pointpillars_detect.npz: the UNMODIFIED reference Anchor3DHead.get_bboxes on the
seeded synthetic head maps of detect_support.PP_DETECT_CASES, driven through the drop-in boundary exactly as
tests/ref_boundary_cases.py drives the other reference flows (whose command line it reuses).  Run as a script in a
fresh process:

    python tests/ref_detect_case.py [--ops oracle] [--record DIR]

`--ops oracle` binds the CPU oracle (no GPU needed); against the CUDA library the script also runs the fused
get_bboxes and the unmodified PointPillars.inference_end after pointpillars.patch_reference_model.  Prints one JSON
line.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_boundary_cases as rbc  # noqa: E402  (puts the repository root on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from detect_support import PP_DETECT_CASES, pp_detect_maps  # noqa: E402


def run(root, dev):
    """The unmodified Anchor3DHead.get_bboxes (anchors, top-k, decode, multiclass_nms through the boundary's nms) on
    seeded synthetic head maps of the KITTI and Waymo heads: a 6 x 5 map with fewer rows than nms_pre, and a class
    with nothing above score_thr.  Against a GPU library, also the fused get_bboxes, and the unmodified
    PointPillars.inference_end after patch_reference_model."""
    import importlib
    from open3d_ml_b200.pointpillars import cfg_from_reference
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    pp_mod = importlib.import_module(ml3d.models.PointPillars.__module__)
    cfgs = {k: Config.load_from_file(os.path.join(root, "ml3d", "configs", "pointpillars_%s.yml" % k))
            for k in ("kitti", "waymo")}
    for k, c in cfgs.items():
        rbc.REC["cfg_" + k] = json.dumps(cfg_from_reference(c.model))
    rbc.REC["cases"] = json.dumps(PP_DETECT_CASES)
    out = dict(boxes_per_frame={})
    for case in PP_DETECT_CASES:
        model_cfg = cfgs[case["head"]].model
        head = pp_mod.Anchor3DHead(num_classes=len(model_cfg["classes"]), **model_cfg["head"]).eval()
        C, A = head.num_classes, head.num_anchors
        maps = [pp_detect_maps(s, case["H"], case["W"], C, A, model_cfg["head"]["rotations"],
                               float(model_cfg["head"].get("dir_offset", 0)), case["n_fg"], case["empty_classes"])
                for s in case["seeds"]]
        cls, reg, dir_ = (torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3))
        with torch.no_grad():
            boxes, scores, labels = head.get_bboxes(cls, reg, dir_)
        out["boxes_per_frame"][case["name"]] = [len(b) for b in boxes]
        for b in range(len(boxes)):
            key = "%s_%d_" % (case["name"], b)
            rbc.REC[key + "boxes"] = boxes[b].numpy()
            rbc.REC[key + "scores"] = scores[b].numpy()
            rbc.REC[key + "labels"] = labels[b].numpy()
        if dev != "cpu":
            from types import SimpleNamespace
            from oracle import weights
            from open3d_ml_b200.pointpillars import patch_reference_model
            net = ml3d.models.PointPillars(**model_cfg, device=dev)
            net.eval()
            man = weights.manifest_from_state_dict(net.state_dict())
            net.load_state_dict(weights.seeded_state_dict(man, rbc.SEED), strict=True)
            patch_reference_model(net)
            maps_d = [t.to(dev) for t in (cls, reg, dir_)]
            got = net.bbox_head.get_bboxes(*maps_d)
            res = net.inference_end(maps_d, SimpleNamespace(calib=[None] * len(boxes)))
            out.setdefault("fused", {})[case["name"]] = dict(
                counts=[len(g) for g in got[0]],
                labels_equal=all(torch.equal(g.cpu(), r) for g, r in zip(got[2], labels)),
                box_err=max([float((g.cpu() - r).abs().max()) for g, r in zip(got[0], boxes) if len(r)] + [0.0]),
                inference_end_counts=[len(r) for r in res],
                inference_end_names=[[bb.label_class for bb in r[:3]] for r in res])
    rbc.record("boundary_pointpillars_detect.npz")
    return out


if __name__ == "__main__":
    rbc.main("pointpillars_detect", run)
