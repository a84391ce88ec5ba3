"""Row (b) of SURVEY.md section 8: the fused forwards against the UNMODIFIED reference classes, on the inputs the
reference's own preprocess / transform / batcher built through the drop-in boundary (open3d_ml_b200.shim /
oracle/refshim.py).  The reference side is stored in tests/golden/boundary_<case>.npz by
`python tests/ref_boundary_cases.py <case> --ops oracle --record tests/golden` where an Open3D-ML tree is available:
the weight manifest (the weights are rebuilt here from it and a seed), those inputs and a seeded sample of the
reference outputs."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import weights

pytestmark = pytest.mark.gpu
TOL = 1e-4


def load(case):
    g = np.load(os.path.join(GOLDEN, "boundary_%s.npz" % case))
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), int(g["weight_seed"]))
    return g, sd


def levels(g, key):
    out, i = [], 0
    while "%s_%d" % (key, i) in g:
        a = torch.from_numpy(g["%s_%d" % (key, i)])
        out.append(a.long() if a.dtype == torch.int32 else a)
        i += 1
    return out


def sampled_rel_err(got, g, name):
    """max |got - ref| over the stored sample of `name`, relative to max |ref| over the whole reference tensor."""
    assert list(got.shape) == g[name + "_shape"].tolist()
    a = got.detach().double().cpu().reshape(-1)[torch.from_numpy(g[name + "_idx"])]
    return float((a - torch.from_numpy(g[name + "_val"])).abs().max() / float(g[name + "_absmax"]))


def test_unmodified_pointpillars_class_matches_fused_forward():
    import open3d_ml_b200 as M
    g, sd = load("pointpillars_class")
    fused = M.PointPillarsB200(sd, json.loads(str(g["cfg"])))
    got = fused([torch.from_numpy(g["point_%d" % i]).cuda() for i in range(int(g["frames"]))])
    assert [g["ref_%d_shape" % i].tolist() for i in range(3)] == [[2, 18, 248, 216], [2, 42, 248, 216], [2, 12, 248, 216]]
    errs = [sampled_rel_err(t, g, "ref_%d" % i) for i, t in enumerate(got)]
    assert all(e < TOL for e in errs), errs


def test_patch_reference_model_randlanet_matches_the_cpu_class():
    from open3d_ml_b200.randlanet import RandLANetB200
    g, sd = load("randlanet_patch")
    fused = RandLANetB200(sd, int(g["num_layers"]), int(g["num_neighbors"]),
                          sub_sampling_ratio=g["sub_sampling_ratio"].tolist())
    inp = {k: levels(g, k) for k in ("coords", "neighbor_indices", "sub_idx", "interp_idx")}
    inp["features"] = torch.from_numpy(g["features"])
    got = fused(inp)
    assert g["ref_shape"].tolist() == [1, 8192, 19]
    err = sampled_rel_err(got, g, "ref")
    agree = float((got.argmax(-1).cpu().reshape(-1) == torch.from_numpy(g["ref_argmax"]).long().reshape(-1)).float().mean())
    assert err < TOL and agree > 0.999, (err, agree)


def test_unmodified_kpfcnn_class_matches_fused_forward():
    import open3d_ml_b200 as M
    g, sd = load("kpconv_class")
    fused = M.KPFCNNB200(sd, json.loads(str(g["cfg"])))
    batch = {k: levels(g, k) for k in ("points", "neighbors", "pools", "upsamples")}
    batch["features"] = torch.from_numpy(g["features"])
    got = fused(batch)
    assert batch["points"][0].shape[0] >= 1000 and g["ref_shape"].tolist()[1] == 5
    err = sampled_rel_err(got, g, "ref")
    assert err < TOL, err
