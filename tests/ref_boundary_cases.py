"""Drives UNMODIFIED reference code (models, dataloaders, pipelines, its own smoke tests) through the
drop-in boundary open3d_ml_b200.shim.  Run as a script in a fresh process (the shim owns
sys.modules['open3d']):

    python tests/ref_boundary_cases.py <case> [--ops oracle] [--record DIR]

`--ops oracle` binds the CPU oracle instead of the CUDA library (oracle/refshim.py): the same flows on a machine
without a GPU.  The models get seeded weights rebuilt from a manifest (oracle/weights.py), so that
`--record DIR` can store what a fused forward needs to be compared without the reference tree: the manifest,
the inputs the reference's own preprocess / transform / batcher built, and a seeded sample of the reference
outputs, as DIR/boundary_<case>.npz (tests/golden/, read by tests/test_gpu_reference_boundary.py).
Prints one JSON line.
"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def install(ops):
    """Binds the CUDA library (`ops` "b200") or the CPU oracle ("oracle") under the reference tree.  -> its root."""
    from oracle.make_ref_snapshot import ref_root
    root = ref_root()
    if root is None:
        print(json.dumps(dict(skipped="no reference tree (neither /root/reference nor oracle/_ref)")))
        sys.exit(0)
    if ops == "oracle":
        from oracle import refshim
        refshim.install()
    else:
        from open3d_ml_b200 import shim
        shim.install(root)
    return root


SEED = 1234
REC = {}          # arrays of the case for --record
RECORD = None     # --record DIR


def seed_weights(net):
    """Seeded weights with non-trivial BN statistics, rebuilt from a manifest of the class's state_dict."""
    from oracle import weights
    man = weights.manifest_from_state_dict(net.state_dict())
    net.load_state_dict(weights.seeded_state_dict(man, SEED), strict=True)
    REC.update(manifest=json.dumps(man), weight_seed=SEED)


def record_output(name, t, m=8192):
    """A fixed, seeded sample of a reference output: flat indices, values, shape and the scale max |t|."""
    a = torch.as_tensor(t).detach().double().cpu().reshape(-1).numpy()
    idx = np.sort(np.random.default_rng(len(REC)).choice(a.size, size=min(m, a.size), replace=False))
    REC.update({name + "_idx": idx.astype(np.int64), name + "_val": a[idx], name + "_shape": np.array(list(t.shape)),
                name + "_absmax": np.abs(a).max()})


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def case_ref_tests(root, dev):
    """The reference's own torch smoke tests (tests/test_models.py:34-73,117-153,204-236), unmodified."""
    import pytest
    os.environ["PATH_TO_OPEN3D_ML"] = root
    os.chdir(tempfile.mkdtemp())          # KPFCNN writes kernels/dispositions/*.npy into the CWD (kpconv.py:1909-1999)
    rc = pytest.main([os.path.join(root, "tests", "test_models.py"), "-q", "-k", "torch", "-p", "no:cacheprovider"])
    return dict(pytest_rc=int(rc))


def case_pointpillars_class(root, dev):
    """Unmodified PointPillars (its own torch layers) fed by the shim's voxelize / ragged_to_dense, against the
    fused PointPillarsB200 built from the same state_dict; then inference_end (anchors, top-k, decode, rotated
    NMS through the shim's nms)."""
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    from open3d_ml_b200 import synth
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "pointpillars_kitti.yml"))
    torch.manual_seed(0)
    net = ml3d.models.PointPillars(**cfg.model, device=dev)
    net.eval()
    seed_weights(net)
    batcher = ml3d.dataloaders.ConcatBatcher(dev, model="PointPillars")
    items = []
    for s in (11, 12):
        d = {"point": synth.lidar_frame(20000, s), "calib": None, "bounding_boxes": []}
        d = net.transform(net.preprocess(d, {"split": "test"}), {"split": "test"})
        items.append({"data": d, "attr": {"split": "test"}})
    data = batcher.collate_fn(items)
    data.to(dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with torch.no_grad():
        ref = net(data)
        boxes = net.inference_end(ref, data)
    out = dict(ref_shapes=[list(r.shape) for r in ref], boxes_per_frame=[len(b) for b in boxes])
    from open3d_ml_b200.pointpillars import cfg_from_reference
    REC.update(cfg=json.dumps(cfg_from_reference(cfg.model)), frames=len(data.point))
    for i, pt in enumerate(data.point):
        REC["point_%d" % i] = pt.detach().cpu().numpy()
    for i, r in enumerate(ref):
        record_output("ref_%d" % i, r)
    if dev != "cpu":
        import open3d_ml_b200 as M
        fused = M.PointPillarsB200(net.state_dict(), cfg_from_reference(cfg.model))
        got = fused(data.point)
        out["rel_err"] = [rel(g, r) for g, r in zip(got, ref)]
    return out


def _randla_inputs(net, n, seed):
    rng = np.random.default_rng(seed)
    from open3d_ml_b200 import synth
    pc = synth.semantickitti_cloud(n, seed)
    data = {"point": pc, "feat": None, "label": rng.integers(0, 19, n).astype(np.int32)}
    attr = {"split": "test"}
    data = net.preprocess(data, attr)
    inp = net.transform(data, attr)
    return {k: ([torch.from_numpy(np.array([a])) for a in v] if isinstance(v, list) else torch.from_numpy(np.array([v])))
            for k, v in inp.items() if k in ("coords", "neighbor_indices", "sub_idx", "interp_idx", "features")}


def case_randlanet_patch(root, dev):
    """patch_reference_model(RandLANet): the unmodified class with its forward on the fused CUDA path, against the
    same class on the CPU; inputs come from the class's own preprocess / transform (k-NN through the shim)."""
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "randlanet_semantickitti.yml"))
    cfg.model["num_points"] = 8192
    torch.manual_seed(0)
    net = ml3d.models.RandLANet(**cfg.model)
    net.device = "cpu"
    net.eval()
    seed_weights(net)
    inp = _randla_inputs(net, 8192, 21)
    with torch.no_grad():
        ref = net(inp)
    out = dict(ref_shape=list(ref.shape))
    REC.update(num_layers=net.cfg.num_layers, num_neighbors=net.cfg.num_neighbors,
               sub_sampling_ratio=np.array(list(net.cfg.sub_sampling_ratio)), features=inp["features"].numpy(),
               ref_argmax=ref.argmax(-1).numpy().astype(np.uint8))
    for k in ("coords", "neighbor_indices", "sub_idx", "interp_idx"):
        for i, a in enumerate(inp[k]):
            a = a.numpy()
            REC["%s_%d" % (k, i)] = a.astype(np.int32) if a.dtype == np.int64 else a
    record_output("ref", ref)
    if dev != "cpu":
        from open3d_ml_b200.randlanet import patch_reference_model
        patch_reference_model(net)
        got = net(inp)
        out["rel_err"] = rel(got, ref)
        out["argmax_agree"] = float((got.argmax(-1).cpu() == ref.argmax(-1)).float().mean())
    return out


def case_semseg_inference(root, dev):
    """SemanticSegmentation.run_inference (semantic_segmentation.py:122-187) on a 20 000-point synthetic cloud,
    unmodified pipeline + dataloader + sampler; natives used: subsample x2, NearestNeighborSearch / knn_search."""
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    from open3d_ml_b200 import synth
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "randlanet_semantickitti.yml"))
    cfg.model["num_points"] = 4096
    torch.manual_seed(0)
    net = ml3d.models.RandLANet(**cfg.model)
    pipe = ml3d.pipelines.SemanticSegmentation(net, dataset=None, device=dev, **cfg.pipeline)
    rng = np.random.default_rng(5)
    pc = synth.semantickitti_cloud(20000, 31)
    data = {"point": pc, "feat": None, "label": rng.integers(1, 19, 20000).astype(np.int32)}
    res = pipe.run_inference(data)
    lab, sc = np.asarray(res["predict_labels"]), np.asarray(res["predict_scores"])
    out = dict(labels_shape=list(lab.shape), scores_shape=list(sc.shape), finite=bool(np.isfinite(sc).all()))
    if dev != "cpu":
        from open3d_ml_b200.randlanet import patch_reference_model
        patch_reference_model(net)           # same pipeline, forward on the fused kernels
        pipe2 = ml3d.pipelines.SemanticSegmentation(net, dataset=None, device=dev, **cfg.pipeline)
        res2 = pipe2.run_inference(data)
        out["fused_labels_shape"] = list(np.asarray(res2["predict_labels"]).shape)
        out["fused_finite"] = bool(np.isfinite(np.asarray(res2["predict_scores"])).all())
    return out


def case_kpconv_class(root, dev):
    """Unmodified KPFCNN (eval) on a batch built by its own preprocess / transform / ConcatBatcher (grid subsampling
    and the 13 radius searches through the shim), against KPFCNNB200 from the same state_dict and batch."""
    import open3d.ml.torch as ml3d
    from open3d_ml_b200 import synth
    os.chdir(tempfile.mkdtemp())
    np.random.seed(3)
    torch.manual_seed(0)
    net = ml3d.models.KPFCNN(lbl_values=[0, 1, 2, 3, 4, 5], num_classes=4, ignored_label_inds=[0], in_features_dim=5,
                             first_subsampling_dl=0.04, in_radius=1.5, min_in_points=3000)
    net.device = "cpu"
    net.eval()
    seed_weights(net)
    pts, feats = synth.room_cloud(6000, 41, room=(2.0, 1.6, 1.2))
    data = {"point": pts, "feat": feats[:, 1:4], "label": np.random.randint(0, 5, len(pts)).astype(np.int32)}
    attr = {"split": "test"}
    batcher = ml3d.dataloaders.ConcatBatcher("cpu")
    data = net.preprocess(data, attr)
    inputs = batcher.collate_fn([{"data": net.transform(data, attr), "attr": attr}])
    with torch.no_grad():
        ref = net(inputs["data"])
    out = dict(ref_shape=list(ref.shape), levels=[int(p.shape[0]) for p in inputs["data"].points])
    b = inputs["data"]
    REC.update(cfg=json.dumps(dict(net.cfg), default=lambda o: o.tolist() if hasattr(o, "tolist") else list(o)),
               levels=len(b.points), features=b.features.numpy())
    for k in ("points", "neighbors", "pools", "upsamples"):
        for i, a in enumerate(getattr(b, k)):
            a = a.numpy()
            REC["%s_%d" % (k, i)] = a.astype(np.int32) if a.dtype == np.int64 else a
    record_output("ref", ref)
    if dev != "cpu":
        import open3d_ml_b200 as M
        fused = M.KPFCNNB200(net.state_dict(), dict(net.cfg))
        got = fused(inputs["data"])
        out["rel_err"] = rel(got, ref)
    return out


def record(name):
    """Writes REC to DIR/name under --record DIR."""
    if RECORD is not None:
        np.savez_compressed(os.path.join(RECORD, name), **REC)


def main(case, run):
    """The recorders' command line: binds the ops `--ops` names, runs run(root, device) and prints its RESULT line."""
    global RECORD
    ops = "oracle" if "--ops" in sys.argv and sys.argv[sys.argv.index("--ops") + 1] == "oracle" else "b200"
    if "--record" in sys.argv:
        RECORD = sys.argv[sys.argv.index("--record") + 1]
    root = install(ops)
    dev = "cpu" if ops == "oracle" or not torch.cuda.is_available() else "cuda"
    res = run(root, dev)
    print("RESULT " + json.dumps(dict(case=case, ops=ops, device=dev, **res)))


CASES = dict(ref_tests=case_ref_tests, pointpillars_class=case_pointpillars_class, randlanet_patch=case_randlanet_patch,
             semseg_inference=case_semseg_inference, kpconv_class=case_kpconv_class)

if __name__ == "__main__":
    case = sys.argv[1]

    def run(root, dev):
        res = CASES[case](root, dev)
        record("boundary_%s.npz" % case)
        return res
    main(case, run)
