"""Drives an UNMODIFIED reference KPFCNN through kpconv.patch_reference_model, in a fresh process (the shim owns
sys.modules['open3d']):

    python tests/kpconv_patch_cases.py <case> [<case> ...] [--ops oracle]

Cases (tests/test_gpu_patch_kpconv.py reads their RESULT lines):
  parity_s3dis, parity_parislille3d  one batch from the reference's own preprocess / transform / ConcatBatcher
                                     (seeded np.random, seeded manifest weights, eval), the unpatched class on the GPU
                                     against the same instance after patch_reference_model
  flow                               SemanticSegmentation.run_inference on a small room, unpatched then patched
  refusals                           train() mode, a modulated deformable config, load_state_dict after patching
`--ops oracle` binds the CPU oracle and runs only the reference side (no GPU needed).  Prints one JSON line per case.
"""
import copy
import json
import os
import random
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_boundary_cases as rbc  # noqa: E402  (puts the repository root on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def model_cfg(root, name, **over):
    from open3d.ml.utils import Config
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", name))
    return dict(cfg.model, **over), cfg.pipeline


# min_in_points: SemSegRandomSampler's sphere takes that many nearest points (the reference default is 3)
S3DIS = ("kpconv_s3dis.yml", dict(min_in_points=8000))
# as tests/ref_kpconv_deform_case.py: a 2 m sphere keeps the deformable batch near 4 000 points
PARIS = ("kpconv_parislille3d.yml", dict(in_radius=2.0, max_in_points=4000, min_in_points=4000, batch_limit=4000))


def seeded_model(root, which, **over):
    import open3d.ml.torch as ml3d
    name, base = which
    mc, pipe = model_cfg(root, name, **dict(base, **over))
    torch.manual_seed(0)
    net = ml3d.models.KPFCNN(**mc)
    net.eval()
    rbc.seed_weights(net)
    return net, pipe


def one_batch(net, pts, feat, label, device):
    """The reference's preprocess / transform / ConcatBatcher.collate_fn, as SemanticSegmentation runs them."""
    import open3d.ml.torch as ml3d
    attr = {"split": "test"}
    data = net.preprocess({"point": pts, "feat": feat, "label": label}, attr)
    items = [{"data": net.transform(data, attr), "attr": attr}]
    return ml3d.dataloaders.ConcatBatcher(device).collate_fn(items)["data"]


def parity(root, dev, which, cloud):
    """The unpatched class on `dev`, then the same instance patched, on the batch as the batcher left it on the CPU
    and after KPConvBatch.to(dev)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    net, _ = seeded_model(root, which)
    np.random.seed(3)
    pts, feat, label = cloud
    b = one_batch(net, pts, feat, label, "cpu")
    on_host = copy.copy(b)                   # KPConvBatch.to rebinds its attributes, the copy keeps the host tensors
    b.to(dev)
    net.to(dev)
    net.device = dev
    with torch.no_grad():
        ref = net(b)
    out = dict(ref_shape=list(ref.shape), levels=[int(p.shape[0]) for p in b.points],
               index_dtypes=sorted({str(t.dtype) for t in b.neighbors + b.pools + b.upsamples}),
               deform_blocks=[i for i, blk in enumerate(net.encoder_blocks) if "deform" in blk.block_name])
    if dev == "cpu":
        return out
    from open3d_ml_b200.kpconv import patch_reference_model
    assert patch_reference_model(net) is net
    with torch.no_grad():
        got_dev = net(b)
        got_host = net(on_host)
    out.update(fused_shape=list(got_dev.shape), fused_dtype=str(got_dev.dtype), fused_device=got_dev.device.type,
               rel_err=rbc.rel(got_dev, ref), rel_err_host_batch=rbc.rel(got_host, ref))
    return out


def case_parity_s3dis(root, dev):
    from open3d_ml_b200 import synth
    pts, feats = synth.room_cloud(12000, 41, room=(3.0, 2.5, 1.5))
    label = np.random.default_rng(4).integers(0, 13, len(pts)).astype(np.int32)
    return parity(root, dev, S3DIS, (pts, feats[:, 1:4] * 255, label))


def case_parity_parislille3d(root, dev):
    from open3d_ml_b200 import synth
    pts = synth.semantickitti_cloud(60000, 51)
    label = np.random.default_rng(5).integers(0, 9, len(pts)).astype(np.int32)
    return parity(root, dev, PARIS, (pts, None, label))


def case_flow(root, dev):
    """SemanticSegmentation.run_inference (semantic_segmentation.py:122-187): spatially regular sampler, the
    reference batcher through the shim, update_probs; unpatched and patched from the same seeds."""
    import open3d.ml.torch as ml3d
    from open3d_ml_b200 import synth
    net, pipe_cfg = seeded_model(root, ("kpconv_s3dis.yml", {}))
    calls = []
    net.register_forward_hook(lambda m, a, o: calls.append(int(o.shape[0])))
    pts, feats = synth.room_cloud(6000, 43, room=(4.0, 3.0, 1.5))
    data = {"point": pts, "feat": feats[:, 1:4] * 255,
            "label": np.random.default_rng(6).integers(0, 13, len(pts)).astype(np.int32)}

    def run():
        np.random.seed(8)
        random.seed(8)
        torch.manual_seed(8)
        pipe = ml3d.pipelines.SemanticSegmentation(net, dataset=None, device=dev, **pipe_cfg)
        res = pipe.run_inference(data)
        return np.asarray(res["predict_labels"]), np.asarray(res["predict_scores"])

    lab, sc = run()
    out = dict(n=len(pts), labels_shape=list(lab.shape), scores_shape=list(sc.shape), batch_points=list(calls))
    calls.clear()
    if dev == "cpu":
        return out
    from open3d_ml_b200.kpconv import patch_reference_model
    patch_reference_model(net)
    flab, fsc = run()
    out.update(fused_batch_points=calls, fused_labels_shape=list(flab.shape), fused_scores_shape=list(fsc.shape),
               fused_finite=bool(np.isfinite(fsc.astype(np.float32)).all()),
               label_agreement=float((flab == lab).mean()),
               score_max_diff=float(np.abs(fsc.astype(np.float32) - sc.astype(np.float32)).max()))
    return out


def case_refusals(root, dev):
    net, _ = seeded_model(root, S3DIS)
    out = {}
    if dev == "cpu":
        return out
    from open3d_ml_b200.kpconv import patch_reference_model
    patch_reference_model(net)
    patched = net.forward
    net.train()
    try:
        net(None)
        out["train_error"] = None
    except RuntimeError as e:
        out["train_error"] = str(e)
    net.eval()
    keys = sorted(net.state_dict())
    net.load_state_dict(net.state_dict(), strict=True)
    out.update(keys_unchanged=sorted(net.state_dict()) == keys, forward_still_patched=net.forward is patched)

    mod, _ = seeded_model(root, PARIS, modulated=True)
    before = mod.forward
    try:
        patch_reference_model(mod)
        out["modulated_error"] = None
    except RuntimeError as e:
        out["modulated_error"] = str(e)
    out["modulated_forward_untouched"] = "forward" not in vars(mod) and mod.forward == before
    return out


CASES = dict(parity_s3dis=case_parity_s3dis, parity_parislille3d=case_parity_parislille3d, flow=case_flow,
             refusals=case_refusals)

if __name__ == "__main__":
    cases = [a for a in sys.argv[1:] if a in CASES]
    os.chdir(tempfile.mkdtemp())          # KPFCNN writes kernels/dispositions/*.npy, the pipeline ./logs, into the CWD

    def run(root, dev):
        # one process for every case: the shim is installed once, and the torch / reference imports are paid once
        for case in cases[:-1]:
            print("RESULT " + json.dumps(dict(case=case, device=dev, **CASES[case](root, dev))), flush=True)
        return CASES[cases[-1]](root, dev)
    rbc.main(cases[-1], run)
