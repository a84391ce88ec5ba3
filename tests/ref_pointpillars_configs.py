"""Records tests/golden/pointpillars_config_<k>.npz for k in nuscenes, argoverse, lyft: the UNMODIFIED reference
PointPillars built from its yml (nuScenes and Argoverse with a two-layer PillarFeatureNet) with seeded weights, and
the unmodified Anchor3DHead.get_bboxes of its head on seeded head maps, driven through the drop-in boundary exactly
as tests/ref_boundary_cases.py drives the other reference flows (whose install / ref_modules / seed_weights /
record_output it reuses).  Run as a script in a fresh process:

    python tests/ref_pointpillars_configs.py [--ops oracle] [--record DIR]

Each fixture holds the manifest (the weights are rebuilt from it and weight_seed), cfg (cfg_from_reference of the
yml), the frames the class's own preprocess / transform / ConcatBatcher built, as the row mask of the seeded
synthetic frame that preprocess kept (point_<i>_kept, bit-packed) and the SHA-256 of the batcher's points
(point_<i>_sha256; pp_configs_support.load regenerates them and checks it), a seeded sample of its three head maps
(ref_<i>) and, per case of pp_configs_support.DETECT_CASES on its head, the reference get_bboxes output per frame
(det_<case>_<b>_boxes / _scores / _labels).  Against the CUDA library the script also prints the fused forward's error.
Prints one JSON line.
"""
import importlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_boundary_cases as rbc  # noqa: E402  (puts the repository root on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from detect_support import pp_detect_maps  # noqa: E402
from pp_configs_support import CONFIGS, DETECT_CASES, digest, fixture, synth_frame  # noqa: E402


def run(root, dev, record_dir=None):
    from open3d_ml_b200.pointpillars import cfg_from_reference
    ml3d, Config = rbc.ref_modules()
    pp_mod = importlib.import_module(ml3d.models.PointPillars.__module__)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = dict(configs={}, boxes_per_frame={})
    for k, spec in CONFIGS.items():
        rbc.REC.clear()
        cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", spec["yml"]))
        torch.manual_seed(0)
        net = ml3d.models.PointPillars(**cfg.model, device=dev)
        net.eval()
        rbc.seed_weights(net)
        batcher = ml3d.dataloaders.ConcatBatcher(dev, model="PointPillars")
        rng = cfg.model["point_cloud_range"]
        items, synth_frames = [], []
        for i in range(len(spec["seeds"])):
            pts = synth_frame(k, i, rng)
            synth_frames.append(pts)
            d = {"point": pts, "calib": None, "bounding_boxes": []}
            d = net.transform(net.preprocess(d, {"split": "test"}), {"split": "test"})
            items.append({"data": d, "attr": {"split": "test"}})
        data = batcher.collate_fn(items)
        data.to(dev)
        with torch.no_grad():
            ref = net(data)
        fcfg = cfg_from_reference(cfg.model)
        rbc.REC.update(cfg=json.dumps(fcfg), frames=len(data.point))
        for i, (pt, pts) in enumerate(zip(data.point, synth_frames)):
            # the rows preprocess keeps (point_pillars.py:218-226); the fixture stores the mask, not the points
            lo, hi = np.array(rng[:3]), np.array(rng[3:])
            kept = np.all((pts[:, :3] >= lo) & (pts[:, :3] < hi), axis=1)
            got = pt.detach().cpu().numpy()
            assert np.array_equal(pts[kept], got), "preprocess kept other rows than the range filter"
            rbc.REC["point_%d_kept" % i] = np.packbits(kept)
            rbc.REC["point_%d_sha256" % i] = digest(got)
        for i, r in enumerate(ref):
            rbc.record_output("ref_%d" % i, r)
        sd = net.state_dict()
        res = dict(pfn=[list(sd["voxel_encoder.pfn_layers.%d.linear.weight" % j].shape)
                        for j in range(len(net.voxel_encoder.pfn_layers))],
                   ref_shapes=[list(r.shape) for r in ref], points=[int(p.shape[0]) for p in data.point])
        if dev != "cpu":
            import open3d_ml_b200 as M
            got = M.PointPillarsB200(sd, fcfg)(data.point)
            res["rel_err"] = [rbc.rel(g, r) for g, r in zip(got, ref)]
        out["configs"][k] = res
        cases = [c for c in DETECT_CASES if c["head"] == k]
        rbc.REC["detect_cases"] = json.dumps(cases)
        head = pp_mod.Anchor3DHead(num_classes=len(cfg.model["classes"]), **cfg.model["head"]).eval()
        for case in cases:
            C, A = head.num_classes, head.num_anchors
            maps = [pp_detect_maps(s, case["H"], case["W"], C, A, cfg.model["head"]["rotations"],
                                   float(cfg.model["head"].get("dir_offset", 0)), case["n_fg"], case["empty_classes"])
                    for s in case["seeds"]]
            cls, reg, dir_ = (torch.from_numpy(np.stack([m[i] for m in maps])) for i in range(3))
            with torch.no_grad():
                boxes, scores, labels = head.get_bboxes(cls, reg, dir_)
            out["boxes_per_frame"][case["name"]] = [len(b) for b in boxes]
            for b in range(len(boxes)):
                key = "det_%s_%d_" % (case["name"], b)
                rbc.REC[key + "boxes"] = boxes[b].numpy()
                rbc.REC[key + "scores"] = scores[b].numpy()
                rbc.REC[key + "labels"] = labels[b].numpy()
        if record_dir is not None:
            np.savez_compressed(os.path.join(record_dir, os.path.basename(fixture(k))), **rbc.REC)
    return out


if __name__ == "__main__":
    rbc.OPS = ops = "oracle" if "--ops" in sys.argv and sys.argv[sys.argv.index("--ops") + 1] == "oracle" else "b200"
    root = rbc.install(ops)
    dev = "cpu" if ops == "oracle" or not torch.cuda.is_available() else "cuda"
    res = run(root, dev, sys.argv[sys.argv.index("--record") + 1] if "--record" in sys.argv else None)
    print("RESULT " + json.dumps(dict(case="pointpillars_configs", ops=ops, device=dev, **res)))
