"""Deformable KPConv without a GPU: the torch port (oracle/models_torch.py) against the unmodified reference's
outputs stored in tests/golden/boundary_kpconv_deform_class.npz (Paris-Lille3D config, recorded by
tests/ref_kpconv_deform_case.py), the tied-kernel-point rule, and kpconv.layer_radii against the radii
KPConvBatch.segmentation_inputs picks (concat_batcher.py:209-262)."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import models_torch as MT, weights
from open3d_ml_b200.kpconv import layer_radii

# largest error of the port against the reference on this fixture: 2.6e-6 (logits), 2.7e-6 (blocks)
TOL = 1e-5


def fixture():
    g = np.load(os.path.join(GOLDEN, "boundary_kpconv_deform_class.npz"))
    sd = weights.seeded_state_dict(json.loads(str(g["manifest"])), int(g["weight_seed"]))
    batch = dict(features=torch.from_numpy(g["features"]))
    for k in ("points", "neighbors", "pools", "upsamples"):
        batch[k] = [torch.from_numpy(g["%s_%d" % (k, i)]) for i in range(int(g["levels"]))]
        batch[k] = [a.long() if a.dtype == torch.int32 else a for a in batch[k]]
    return g, sd, batch, json.loads(str(g["cfg"]))


def sampled_rel_err(got, g, name):
    assert list(got.shape) == g[name + "_shape"].tolist()
    a = got.detach().double().cpu().reshape(-1)[torch.from_numpy(g[name + "_idx"])]
    return float((a - torch.from_numpy(g[name + "_val"])).abs().max() / float(g[name + "_absmax"]))


@pytest.fixture(scope="module")
def port():
    g, sd, batch, cfg = fixture()
    taps, stats = {}, {}
    with torch.no_grad():
        out = MT.kpfcnn_forward(sd, batch, cfg, taps=taps, stats=stats)
    return g, out, taps, stats


def test_port_reproduces_the_reference_fixture(port):
    g, out, taps, _ = port
    assert g["deform_blocks"].tolist() == [5, 6, 7, 8, 9]
    errs = {"ref": sampled_rel_err(out, g, "ref")}
    for i in g["deform_blocks"].tolist():
        errs[i] = sampled_rel_err(taps["encoder_blocks.%d" % i], g, "enc_%d" % i)
    assert max(errs.values()) < TOL, errs


def test_every_deformable_conv_keeps_and_drops_with_real_offsets(port):
    _, _, _, stats = port
    assert len(stats) == 5
    for name, s in stats.items():
        assert s["kept"] > 0 and s["dropped"] > 0, (name, s)
        assert s["median_offset"] > 0.1, (name, s)        # median |offset| / extent: 2.3-3.4 on this fixture


def test_port_follows_offset_conv_kernel_points():
    g, sd, batch, cfg = fixture()
    p = "encoder_blocks.5.KPConv"
    assert not torch.equal(sd[p + ".kernel_points"], sd[p + ".offset_conv.kernel_points"])   # seeded apart
    base = {}
    with torch.no_grad():
        MT.kpfcnn_forward(sd, batch, cfg, taps=base)
        other = dict(sd)
        other[p + ".kernel_points"] = sd[p + ".kernel_points"] * 3.0 + 1.0
        moved = {}
        MT.kpfcnn_forward(other, batch, cfg, taps=moved)
        assert torch.equal(moved["encoder_blocks.5"], base["encoder_blocks.5"])
        swapped = dict(sd)
        swapped[p + ".offset_conv.kernel_points"] = sd[p + ".kernel_points"]
        MT.kpfcnn_forward(swapped, batch, cfg, taps=moved)
        assert not torch.allclose(moved["encoder_blocks.5"], base["encoder_blocks.5"])


PARIS_ARCH = ["simple", "resnetb", "resnetb_strided", "resnetb", "resnetb_strided", "resnetb_deformable",
              "resnetb_deformable_strided", "resnetb_deformable", "resnetb_deformable_strided", "resnetb_deformable",
              "nearest_upsample", "unary", "nearest_upsample", "unary", "nearest_upsample", "unary",
              "nearest_upsample", "unary"]


def test_layer_radii_paris_lille3d():
    cfg = dict(architecture=PARIS_ARCH, first_subsampling_dl=0.08, conv_radius=2.5, deform_radius=6.0)
    # r = 0.2, 0.4, 0.8, 1.6, 3.2; deform radius = r * 6 / 2.5 from layer 2 on (its blocks and closing block are
    # deformable); layer 4 closes with nearest_upsample, so only its conv neighbours use the deform radius
    want = [(0.2, 0.2, 0.4), (0.4, 0.4, 0.8), (1.92, 1.92, 3.84), (3.84, 3.84, 7.68), (7.68, 3.2, 6.4)]
    got = layer_radii(cfg)
    assert len(got) == 5
    for g, w in zip(got, want):
        assert g == pytest.approx(w, rel=1e-12)


def test_layer_radii_rigid_configs_are_unchanged():
    from conftest import GOLDEN
    with open(os.path.join(GOLDEN, "kpconv_s3dis.manifest.json")) as f:
        cfg = json.load(f)["cfg"]
    r, want = cfg["first_subsampling_dl"] * cfg["conv_radius"], []
    for _ in range(cfg["num_layers"]):          # what build_batch used for every config before deform radii
        want.append((r, r, 2 * r))
        r = r * 2
    assert layer_radii(cfg) == want
    assert layer_radii(dict(cfg, deform_radius=6.0)) == want
