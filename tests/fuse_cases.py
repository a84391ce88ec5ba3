"""Drives ``fuse.fuse_reference_models()`` on UNMODIFIED reference instances in a fresh process (the shim owns
sys.modules['open3d']); tests/test_gpu_fuse.py reads its RESULT line.

    python tests/fuse_cases.py
"""
import json
import logging
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_boundary_cases as rbc  # noqa: E402  (puts the repository root on sys.path)
import kpconv_patch_cases as kpc  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402


class _Records(logging.Handler):
    def __init__(self):
        super().__init__(logging.DEBUG)
        self.lines = []

    def emit(self, record):
        self.lines.append((record.levelname, record.getMessage()))


def randlanet_dispatch(root, builds):
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    from open3d_ml_b200.randlanet import fused_from_reference
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "randlanet_semantickitti.yml"))
    cfg.model["num_points"] = 8192
    torch.manual_seed(0)
    net = ml3d.models.RandLANet(**cfg.model)
    net.device = "cpu"
    rbc.seed_weights(net)
    inp = rbc._randla_inputs(net, 8192, 21)
    inp = {k: [t.cuda() for t in v] if isinstance(v, list) else v.cuda() for k, v in inp.items()}
    net.cuda()
    net.device = "cuda"
    out = {}
    # train: the reference forward, bit for bit
    net.train()
    with torch.no_grad():
        torch.manual_seed(5)
        got = net(inp)
        torch.manual_seed(5)
        want = type(net).forward.__wrapped__(net, inp)
    out["train_bits_equal"] = bool(torch.equal(got, want))
    out["train_builds"] = len(builds)
    # eval: the fused forward of the weights held now, built once while they stay
    net.eval()
    first = net(inp)
    again = net(inp)
    out["eval_builds_after_two_calls"] = len(builds)
    out["eval_repeat_equal"] = bool(torch.equal(first, again))
    out["eval_vs_fresh_fused"] = rbc.rel(first, fused_from_reference(net).forward(inp))
    with torch.no_grad():
        ref = type(net).forward.__wrapped__(net, inp)
    out["eval_vs_reference"] = rbc.rel(first, ref)
    # other weights between two eval calls
    from oracle import weights
    net.load_state_dict(weights.seeded_state_dict(weights.manifest_from_state_dict(net.state_dict()), rbc.SEED + 1))
    second = net(inp)
    out["builds_after_load_state_dict"] = len(builds)
    out["second_vs_fresh_fused"] = rbc.rel(second, fused_from_reference(net).forward(inp))
    out["second_vs_first"] = rbc.rel(second, first)
    return out


def kpconv_refused(root):
    from open3d_ml_b200 import synth
    mod, _ = kpc.seeded_model(root, kpc.PARIS, modulated=True)
    pts = synth.semantickitti_cloud(60000, 51)
    label = np.random.default_rng(5).integers(0, 9, len(pts)).astype(np.int32)
    np.random.seed(3)
    b = kpc.one_batch(mod, pts, None, label, "cpu")
    b.to("cuda")
    mod.cuda()
    mod.device = "cuda"
    with torch.no_grad():
        got = mod(b)
        again = mod(b)
        want = type(mod).forward.__wrapped__(mod, b)
    return dict(refused_equal_reference=bool(torch.equal(got, want) and torch.equal(again, want)))


def pointpillars(root):
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    from open3d_ml_b200 import synth
    from open3d_ml_b200.pointpillars import fused_from_reference
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "pointpillars_kitti.yml"))
    torch.manual_seed(0)
    net = ml3d.models.PointPillars(**cfg.model, device="cuda")
    rbc.seed_weights(net)
    net.cuda()
    net.eval()
    batcher = ml3d.dataloaders.ConcatBatcher("cuda", model="PointPillars")
    items = []
    for s in (11, 12):
        d = {"point": synth.lidar_frame(20000, s), "calib": None, "bounding_boxes": []}
        d = net.transform(net.preprocess(d, {"split": "test"}), {"split": "test"})
        items.append({"data": d, "attr": {"split": "test"}})
    data = batcher.collate_fn(items)
    data.to("cuda")
    head = net.bbox_head
    reference = type(head).get_bboxes.__wrapped__
    with torch.no_grad():
        maps = net(data)
        got = head.get_bboxes(*maps)
        want = fused_from_reference(net).get_bboxes(*maps)
        out = dict(eval_fused_decode=all(torch.equal(a, b) for x, y in zip(got, want) for a, b in zip(x, y)),
                   eval_boxes=[int(len(b)) for b in got[0]])
        net.train()
        tmaps = [m.detach() for m in maps]
        got_t = head.get_bboxes(*tmaps)
        want_t = reference(head, *tmaps)
    out["train_reference_decode"] = all(torch.equal(a, b) for x, y in zip(got_t, want_t) for a, b in zip(x, y))
    return out


def main():
    torch.backends.cuda.matmul.allow_tf32 = False      # the reference forward in float32, as the parity tests run it
    torch.backends.cudnn.allow_tf32 = False
    os.chdir(tempfile.mkdtemp())          # KPFCNN writes its kernel dispositions into the working directory
    root = rbc.install("b200")
    from open3d_ml_b200 import fuse, randlanet
    builds = []
    build = randlanet.fused_from_reference

    def counted(model):
        builds.append(1)
        return build(model)
    randlanet.fused_from_reference = counted
    records = _Records()
    logging.getLogger("open3d_ml_b200.fuse").addHandler(records)
    logging.getLogger("open3d_ml_b200.fuse").setLevel(logging.DEBUG)
    fuse.fuse_reference_models()
    res = dict(randlanet=randlanet_dispatch(root, builds), kpconv=kpconv_refused(root), pointpillars=pointpillars(root))
    res["log"] = records.lines
    print("RESULT " + json.dumps(res))


if __name__ == "__main__":
    main()
