"""Seeded on-disk datasets, configs and checkpoints for the UNMODIFIED ``scripts/run_pipeline.py``, and a driver that
runs it in a fresh process (the shim owns sys.modules['open3d']).

    python tests/run_pipeline_cases.py make <family> <dir> [--scale S]
        writes <dir>/data (the dataset in its own on-disk layout), <dir>/<family>.yml (the shipped yml's model and
        pipeline sections unchanged but for RandLA-Net's in_channels and PointPillars' num_workers, the dataset section pointing at <dir>/data) and <dir>/ckpt.pth
        ({'model_state_dict': seeded weights}); prints one JSON line with the command line arguments to use.
    python tests/run_pipeline_cases.py run <mode> <out> -- <run_pipeline.py arguments>
        seeds the global RNGs, then runs the script in this process:
          launch   as ``python -m open3d_ml_b200.run_pipeline`` does (shim + fused dispatch)
          shim     with the shim alone: the reference forwards
          patched  the shim, and the patch every model module's patch_reference_model makes (fuse.patch) right after
                   the pipeline loaded the checkpoint
          stale    the same patch right before the checkpoint is loaded (after ``model.eval()``), on the init weights
        and stores every result the dataset's save_test_result receives under <out> (labels and scores of each
        cloud, the boxes of each frame).

The datasets are the ones the shipped configs name, in their own layouts: SemanticKITTI sequences, S3DIS
``original_pkl`` rooms, ScanNet ``scene*_vert.npy`` scenes and a KITTI ``testing/`` tree.  (``Custom3D`` cannot hold
test results: its save_test_result indexes a dict with the label array.)
"""
import json
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402

FAMILIES = ("randlanet_semantickitti", "kpconv_s3dis", "pointpillars_kitti", "pvcnn_s3dis", "sparseconvunet_scannet")
WEIGHT_SEED = 1234

# a KITTI calibration (object benchmark layout): P0..P3, R0_rect, Tr_velo_to_cam
_P2 = "7.215377e+02 0 6.095593e+02 4.485728e+01 0 7.215377e+02 1.728540e+02 2.163791e-01 0 0 1 2.745884e-03"
_CALIB = "\n".join(["P0: " + _P2, "P1: " + _P2, "P2: " + _P2, "P3: " + _P2,
                    "R0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 "
                    "7.402527e-03 4.351614e-03 9.999631e-01",
                    "Tr_velo_to_cam: 7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 "
                    "7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01",
                    ""])


def _write_data(family, data, scale):
    """The dataset files of `family` under `data`.  -> {result name: number of points (or 1 per frame)}."""
    from open3d_ml_b200 import synth
    expect = {}
    if family == "randlanet_semantickitti":
        d = os.path.join(data, "dataset", "sequences", "11", "velodyne")
        os.makedirs(d)
        for i in range(scale):
            n = 50000
            p = np.concatenate([synth.semantickitti_cloud(n, 100 + i), np.zeros((n, 1), np.float32)], 1)
            p.astype(np.float32).tofile(os.path.join(d, "%06d.bin" % i))
            os.makedirs(os.path.join(d, "..", "labels"), exist_ok=True)     # raw SemanticKITTI ids, so run_test scores
            np.random.default_rng(700 + i).choice([10, 40, 48, 50, 70, 80], n).astype(np.uint32).tofile(
                os.path.join(d, "..", "labels", "%06d.label" % i))
            expect["11_%06d" % i] = n
    elif family in ("kpconv_s3dis", "pvcnn_s3dis"):
        import pickle
        area = 3 if family == "kpconv_s3dis" else 5
        os.makedirs(os.path.join(data, "original_pkl"))
        for i in range(scale):
            pts, f = synth.room_cloud(40000, 200 + i, room=(5.0, 4.0, 2.7))
            lab = np.random.default_rng(300 + i).integers(0, 13, len(pts))
            pc = np.concatenate([pts, f[:, 1:4] * 255, lab[:, None]], 1).astype(np.float32)
            name = "Area_%d_office_%d" % (area, i + 1)
            with open(os.path.join(data, "original_pkl", name + ".pkl"), "wb") as fh:
                pickle.dump([pc, []], fh)
            expect[name] = len(pts)
        # a training room, so that the tree is not only the test area
        with open(os.path.join(data, "original_pkl", "Area_1_office_1.pkl"), "wb") as fh:
            pickle.dump([pc, []], fh)
    elif family == "sparseconvunet_scannet":
        os.makedirs(data)
        ids = [3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 14, 16, 24, 28, 33, 34, 36, 39]
        for i in range(scale):
            pts, f = synth.room_cloud(60000, 400 + i, dl=0.01, room=(5.0, 4.0, 2.7))
            scene = "scene%04d_00" % (707 + i)        # scannetv2_test.txt lists scene0707_00 onwards
            base = os.path.join(data, scene)
            np.save(base + "_vert.npy", np.concatenate([pts, f[:, 1:4] * 255], 1).astype(np.float32))
            np.save(base + "_sem_label.npy", np.random.default_rng(500 + i).choice(ids, len(pts)).astype(np.int64))
            np.save(base + "_ins_label.npy", np.zeros(len(pts), np.int64))
            np.save(base + "_bbox.npy", np.zeros((0, 7), np.float32))
            expect[scene] = len(pts)
    elif family == "pointpillars_kitti":
        for sub in ("velodyne", "calib"):
            os.makedirs(os.path.join(data, "testing", sub))
        for i in range(scale):
            synth.lidar_frame(60000, 600 + i).tofile(os.path.join(data, "testing", "velodyne", "%06d.bin" % i))
            with open(os.path.join(data, "testing", "calib", "%06d.txt" % i), "w") as fh:
                fh.write(_CALIB)
            expect["%06d" % i] = 1
    else:
        raise KeyError(family)
    return expect


def make(family, out, scale=1):
    """Dataset, config and checkpoint of `family` under `out` (see the module doc)."""
    import yaml
    import torch
    from oracle.make_ref_snapshot import ref_root
    from open3d_ml_b200 import shim
    from oracle import weights
    root = ref_root()
    shim.install(root)
    import open3d.ml.torch as ml3d
    out = os.path.abspath(out)
    os.makedirs(out, exist_ok=True)
    data = os.path.join(out, "data")
    expect = _write_data(family, data, scale)
    with open(os.path.join(root, "ml3d", "configs", family + ".yml")) as fh:
        cfg = yaml.safe_load(fh)
    # no preprocessing cache: the runs of one dataset may be concurrent
    cfg["dataset"].update(dataset_path=data, cache_dir=os.path.join(out, "cache"), use_cache=False,
                          test_result_folder=os.path.join(out, "test"))
    if family == "pvcnn_s3dis":
        # PVCNN.preprocess resamples every cloud to num_points, and the pipeline predicts those points
        expect = {k: cfg["model"]["num_points"] for k in expect}
    if family == "randlanet_semantickitti":
        cfg["dataset"]["test_split"] = ["11"]
        # SemanticKITTI's loader passes the intensity column on as a feature, which the shipped in_channels: 3 refuses
        cfg["model"]["in_channels"] = 4
    if family == "pointpillars_kitti":
        # ObjectDetection.run_test hands its loader workers a lambda, which the script's forkserver cannot pickle
        cfg["pipeline"]["num_workers"] = 0
    path = os.path.join(out, family + ".yml")
    with open(path, "w") as fh:
        yaml.safe_dump(cfg, fh)
    cwd = os.getcwd()
    os.chdir(out)                      # KPFCNN writes its kernel dispositions into the working directory
    try:
        kw = {k: v for k, v in cfg["model"].items() if k != "name"}
        if cfg["model"]["name"] == "PointPillars":
            kw["device"] = "cpu"           # its constructor places the anchors on the device it is given
        model = getattr(ml3d.models, cfg["model"]["name"])(**kw)
    finally:
        os.chdir(cwd)
    sd = weights.seeded_state_dict(weights.manifest_from_state_dict(model.state_dict()), WEIGHT_SEED)
    for k, v in model.state_dict().items():
        if k.endswith(".offset"):
            sd[k] = v.clone()              # SparseConv's lattice offsets stay as constructed
    ckpt = os.path.join(out, "ckpt.pth")
    torch.save({"model_state_dict": sd}, ckpt)
    return dict(family=family, cfg=path, ckpt=ckpt, test=os.path.join(out, "test"), expect=expect,
                args=["torch", "-c", path, "--split", "test", "--ckpt_path", ckpt])


def _record_results(out):
    """Stores what every dataset's save_test_result receives under `out`, then lets it save as it does."""
    import ml3d.datasets as D

    def box_rows(boxes):
        return np.array([list(b.center) + list(b.size) + [float(b.yaw), float(b.confidence)] for b in boxes],
                        np.float64).reshape(-1, 8)

    def wrap(cls):
        save = cls.save_test_result

        def save_test_result(self, results, attr):
            if isinstance(attr, dict):
                np.savez(os.path.join(out, attr["name"] + ".npz"), labels=np.asarray(results["predict_labels"]),
                         scores=np.asarray(results["predict_scores"], np.float32))
            else:
                # ObjectDetectBatch leaves its attr list empty, so KITTI.save_test_result writes no file: the frames
                # are named by their place in the unshuffled test split instead
                for boxes in results:
                    np.savez(os.path.join(out, "%06d.npz" % len(os.listdir(out))), boxes=box_rows(boxes),
                             labels=np.array([b.label_class for b in boxes], dtype=object).astype(str))
            return save(self, results, attr)
        cls.save_test_result = save_test_result
    for name in ("SemanticKITTI", "S3DIS", "Scannet", "KITTI"):
        wrap(getattr(D, name))


def _patch_at_load(after):
    """Patches the model explicitly when the pipeline loads its checkpoint: after loading it or (stale) before."""
    import ml3d.torch.pipelines as P
    from open3d_ml_b200 import fuse

    def patch(model):
        fuse.patch(model, fuse._builders()[type(model).__name__])

    for cls in (P.SemanticSegmentation, P.ObjectDetection):
        load = cls.load_ckpt

        def load_ckpt(self, *a, _load=load, **k):
            if not after:
                patch(self.model)
            r = _load(self, *a, **k)
            if after:
                patch(self.model)
            return r
        cls.load_ckpt = load_ckpt


def run(mode, out, argv):
    import random
    import torch
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    os.makedirs(out, exist_ok=True)
    from open3d_ml_b200 import run_pipeline as RP
    script, rest = RP.prepare(argv)
    _record_results(out)
    if mode == "launch":
        from open3d_ml_b200.fuse import fuse_reference_models
        fuse_reference_models()
    elif mode in ("patched", "stale"):
        _patch_at_load(after=mode == "patched")
    elif mode != "shim":
        raise KeyError(mode)
    sys.argv = [script] + rest
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    if sys.argv[1] == "make":
        scale = int(sys.argv[sys.argv.index("--scale") + 1]) if "--scale" in sys.argv else 1
        print("RESULT " + json.dumps(make(sys.argv[2], sys.argv[3], scale)), flush=True)
    elif sys.argv[1] == "run":
        sep = sys.argv.index("--")
        run(sys.argv[2], sys.argv[3], sys.argv[sep + 1:])
    else:
        raise SystemExit(__doc__)
