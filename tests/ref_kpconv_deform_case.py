"""Records tests/golden/boundary_kpconv_deform_class.npz: the UNMODIFIED reference KPFCNN built from
ml3d/configs/kpconv_parislille3d.yml (deformable layers 2-4, reduce_fc head), on a batch its own preprocess /
transform / ConcatBatcher built through the drop-in boundary (so the neighbourhoods are the deform-radius ones), with
seeded manifest weights.  Reuses tests/ref_boundary_cases.py's command line, seed_weights and record_output.
Run as a script in a fresh process:

    python tests/ref_kpconv_deform_case.py [--ops oracle] [--record DIR]

`--ops oracle` binds the CPU oracle (no GPU needed).  The script asserts that the torch port
(oracle/models_torch.kpfcnn_forward) matches the reference to < 1e-5 on the logits and on every deformable encoder
block; against a GPU library it also runs KPFCNNB200 on the same batch.  Prints one JSON line.
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_boundary_cases as rbc  # noqa: E402  (puts the repository root on sys.path)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import models_torch as MT  # noqa: E402

# a 4 m Paris-Lille3D sphere at 0.08 m has ~10 000 points; these keep the fixture under ~2 MB
IN_RADIUS, MAX_IN_POINTS, BATCH_LIMIT = 2.0, 4000, 4000


def run(root, dev):
    import open3d.ml.torch as ml3d
    from open3d.ml.utils import Config
    from open3d_ml_b200 import synth
    os.chdir(tempfile.mkdtemp())          # KPFCNN writes kernels/dispositions/*.npy into the CWD
    cfg = Config.load_from_file(os.path.join(root, "ml3d", "configs", "kpconv_parislille3d.yml"))
    mc = dict(cfg.model, in_radius=IN_RADIUS, max_in_points=MAX_IN_POINTS, min_in_points=1000,
              batch_limit=BATCH_LIMIT)
    np.random.seed(7)
    torch.manual_seed(0)
    net = ml3d.models.KPFCNN(**mc)
    net.device = "cpu"
    net.eval()
    rbc.seed_weights(net)
    deform = [i for i, b in enumerate(net.encoder_blocks) if "deform" in b.block_name]
    taps = {}
    for i in deform:
        net.encoder_blocks[i].register_forward_hook(lambda m, a, o, i=i: taps.__setitem__(i, o))
    pts = synth.semantickitti_cloud(60000, 51)
    data = {"point": pts, "feat": None, "label": np.random.randint(0, 9, len(pts)).astype(np.int32)}
    attr = {"split": "test"}
    batcher = ml3d.dataloaders.ConcatBatcher("cpu")
    data = net.preprocess(data, attr)
    inputs = batcher.collate_fn([{"data": net.transform(data, attr), "attr": attr}])
    b = inputs["data"]
    with torch.no_grad():
        ref = net(b)
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    bd = dict(features=b.features, points=list(b.points), neighbors=list(b.neighbors), pools=list(b.pools),
              upsamples=list(b.upsamples))
    port_taps, stats = {}, {}
    with torch.no_grad():
        port = MT.kpfcnn_forward(sd, bd, dict(net.cfg), taps=port_taps, stats=stats)
    errs = dict(logits=rbc.rel(port, ref))
    for i in deform:
        errs["encoder_blocks.%d" % i] = rbc.rel(port_taps["encoder_blocks.%d" % i], taps[i])
    assert max(errs.values()) < 1e-5, errs
    out = dict(ref_shape=list(ref.shape), levels=[int(p.shape[0]) for p in b.points],
               widths=[int(n.shape[1]) for n in b.neighbors], deform_blocks=deform, port_rel_err=errs, stats=stats)
    rbc.REC.update(cfg=json.dumps(dict(net.cfg), default=lambda o: o.tolist() if hasattr(o, "tolist") else list(o)),
                   levels=len(b.points), features=b.features.numpy(), deform_blocks=np.array(deform))
    for k in ("points", "neighbors", "pools", "upsamples"):
        for i, a in enumerate(getattr(b, k)):
            a = a.numpy()
            rbc.REC["%s_%d" % (k, i)] = a.astype(np.int32) if a.dtype == np.int64 else a
    rbc.record_output("ref", ref)
    for i in deform:
        rbc.record_output("enc_%d" % i, taps[i], m=4096)
    if dev != "cpu":
        import open3d_ml_b200 as M
        got = M.KPFCNNB200(net.state_dict(), dict(net.cfg))(b)
        out["fused_rel_err"] = rbc.rel(got, ref)
    rbc.record("boundary_kpconv_deform_class.npz")
    return out


if __name__ == "__main__":
    rbc.main("kpconv_deform_class", run)
