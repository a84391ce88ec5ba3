"""The PVCNN kernels and the fused forward against float64: voxel coordinates and cells, the cell mean, the 3x3x3
tensor-core convolution, trilinear devoxelization, and PVCNNB200 against the recorded reference and the torch port."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import open3d_ml_b200 as M
from open3d_ml_b200 import _lib as L, ops, pvcnn, synth
from oracle import pvcnn as PV
from oracle.make_ref_snapshot import ref_root
from conftest import rel_err
import helpers as H
import pvcnn_support as PS
from test_gpu_dense import DENSE_TOL

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


def voxel_cells(pts, r, eps=1e-6):
    """o3dml_pv_voxel_cells on host clouds [B, N, 3] -> (vox [B, N, 3], cell [B, N]) device tensors."""
    B, N, _ = pts.shape
    d = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda().view(B * N, 3)
    stats, vox = torch.empty(B, 4).cuda(), torch.empty(B * N, 3).cuda()
    cell = torch.empty(B * N, dtype=torch.int32).cuda()
    L.check(L.lib().o3dml_pv_voxel_cells(L.ptr(d), B, N, r, eps, L.ptr(stats), L.ptr(vox), L.ptr(cell), L.stream()))
    return vox.view(B, N, 3), cell.view(B, N)


def grouped(cell, num_cells):
    """The points by cell through the library's own invert_neighbors_list: (row splits, point ids)."""
    n = cell.numel()
    res = ops.invert_neighbors_list(num_cells, cell.reshape(-1), torch.arange(n + 1, dtype=torch.int64).cuda(),
                                    torch.empty(0))
    return res.neighbors_row_splits, res.neighbors_index


def clouds(kind, B, N, resolutions, seed=20):
    out = []
    for b in range(B):
        if kind == "room":
            out.append(PS.filtered_cloud(N, seed + b, resolutions)[0])
        else:
            out.append(PV.pv_margin_nudge(synth.uniform_cloud(N, seed + b), resolutions))
    return np.stack(out)


# ---------------------------------------------------------------------------------------------------- cells
@pytest.mark.parametrize("kind", ["room", "uniform"])
@pytest.mark.parametrize("B", [1, 3])
def test_cells_match_the_float64_partition(kind, B):
    res = [1, 2, 24, 32, 64]
    pts = clouds(kind, B, 3000, res)
    for r in res:
        vox, cell = voxel_cells(pts, r)
        v64, c64 = PV.np_pv_voxel_cells(pts, r)
        assert np.array_equal(cell.cpu().numpy(), c64), r
        assert np.abs(vox.cpu().numpy() - v64).max() <= 4 * np.finfo(np.float32).eps * r, r


def test_ties_round_to_even_and_clamp():
    vox, cell = voxel_cells(PS.tie_cloud(), PS.TIE_R, eps=0.0)
    assert np.array_equal(vox[0, :, 0].cpu().numpy(), PS.TIE_VOX_X)
    assert np.array_equal(cell[0].cpu().numpy(), PS.tie_cells())


@pytest.mark.parametrize("n", [1, 7])
def test_identical_points_land_in_the_centre(n):
    vox, cell = voxel_cells(np.full((2, n, 3), 3.25, np.float32), 5)
    assert bool((vox == 2.5).all())
    assert cell.cpu().tolist() == [[62] * n, [187] * n]


# ------------------------------------------------------------------------------------------------ cell mean
def cell_mean(cell, num_cells, feat, cpad):
    splits, ids = grouped(cell, num_cells)
    grid = torch.full((num_cells, cpad), float("nan")).cuda()
    L.check(L.lib().o3dml_pv_cell_mean(L.ptr(splits), L.ptr(ids), num_cells, L.ptr(feat), feat.stride(0),
                                       feat.shape[1], cpad, L.ptr(grid), L.stream()))
    return grid


@pytest.mark.parametrize("C", [9, 64, 128])
def test_cell_mean(C):
    B, N, r = 2, 5000, 16
    pts = clouds("room", B, N, [r])
    _, cell = voxel_cells(pts, r)
    feat = rnd(B * N, C, seed=C)
    cpad = pvcnn.pad32(C)
    grid = cell_mean(cell, B * r ** 3, feat, cpad)
    want = PV.np_avg_voxelize(feat.cpu().numpy().reshape(B, N, C), cell.cpu().numpy(), B * r ** 3)
    got = grid.cpu().numpy()
    assert np.abs(got[:, :C] - want).max() <= 1e-6 * np.abs(want).max()
    empty = np.bincount(cell.cpu().numpy().reshape(-1), minlength=B * r ** 3) == 0
    assert empty.any() and np.all(got[empty] == 0) and np.all(got[:, C:] == 0)
    assert torch.equal(grid, cell_mean(cell, B * r ** 3, feat, cpad))


def test_cell_mean_of_a_cell_holding_every_point():
    n, C = 3000, 9
    _, cell = voxel_cells(np.full((1, n, 3), 1.5, np.float32), 5)       # every coordinate 2.5, which rounds to 2
    feat = rnd(n, C, seed=3)
    grid = cell_mean(cell, 125, feat, 32).cpu().numpy()
    want = feat.cpu().numpy().astype(np.float64).mean(0)
    assert np.abs(grid[62, :C] - want).max() <= 1e-6 * np.abs(feat.cpu().numpy()).max()
    assert np.count_nonzero(grid) == C


# ------------------------------------------------------------------------------------------------ convolution
def conv_case(B, dims, C, Co, epilogue, seed=1):
    X, Y, Z = dims
    x = rnd(B, X, Y, Z, C, seed=seed)
    w = rnd(Co, C, 3, 3, 3, seed=seed + 1) / (27 * C) ** 0.5
    s, t = (rnd(Co, seed=seed + 2).abs() + 0.5, rnd(Co, seed=seed + 3)) if epilogue else (None, None)
    out = torch.full((B, X, Y, Z, Co), float("nan")).cuda()
    wt = L.pack_linear(w.permute(2, 3, 4, 1, 0).reshape(27 * C, Co))
    L.conv3x3x3(x, wt, out, s, t, act="leaky" if epilogue else None, slope=0.1)
    ref = F.conv3d(x.permute(0, 4, 1, 2, 3).double().cpu(), w.double().cpu(), None, 1, 1)
    if epilogue:
        ref = F.leaky_relu(ref * s.double().cpu().view(1, -1, 1, 1, 1) + t.double().cpu().view(1, -1, 1, 1, 1), 0.1)
    return rel_err(out, ref.permute(0, 2, 3, 4, 1))


@pytest.mark.parametrize("epilogue", [False, True])
@pytest.mark.parametrize("dims", [(1, 1, 1), (2, 2, 2), (3, 5, 7), (24, 24, 24)])
@pytest.mark.parametrize("B", [1, 3])
def test_conv3x3x3_small_and_odd_grids(B, dims, epilogue):
    errs = {(C, Co): conv_case(B, dims, C, Co, epilogue, seed=C + Co)
            for C, Co in ((32, 13), (64, 64), (128, 160), (64, 128))}
    assert max(errs.values()) < DENSE_TOL, errs


@pytest.mark.parametrize("C,Co", [(32, 64), (64, 64), (128, 128)])
def test_conv3x3x3_at_32_cubed(C, Co):
    assert conv_case(1, (32, 32, 32), C, Co, True) < DENSE_TOL


def test_conv3x3x3_refuses_channels_off_the_slice_width():
    x, out = rnd(1, 4, 4, 4, 48), torch.empty(1, 4, 4, 4, 16).cuda()
    with pytest.raises(RuntimeError, match="multiple of 32"):
        L.conv3x3x3(x, L.pack_linear(rnd(27 * 48, 16)), out)


# ---------------------------------------------------------------------------------------------- devoxelization
def boundary_vox(B, N, r, seed):
    rng = np.random.default_rng(seed)
    vox = rng.uniform(0, r - 1, (B, N, 3)).astype(np.float32)
    vox[:, :6] = np.array([[0, 0, 0], [r - 1] * 3, [1, 2, r - 1], [r - 1, 0, 0.5], [0.25, r - 1, 0], [2, 2, 2]],
                          np.float32)
    return vox


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("r,C", [(4, 32), (24, 64), (5, 13)])
def test_trilinear_devoxelize(r, C, accumulate):
    B, N, ld = 2, 700, 200
    vox = boundary_vox(B, N, r, r)
    grid = rnd(B * r ** 3, C, seed=r)
    base = rnd(B * N, ld, seed=r + 1)
    out = base.clone()
    inds, wgts = torch.empty(B, 8, N, dtype=torch.int32).cuda(), torch.empty(B, 8, N).cuda()
    dv = torch.from_numpy(vox).cuda().view(B * N, 3)
    L.check(L.lib().o3dml_trilinear_devoxelize(L.ptr(dv), B, N, r, L.ptr(grid), C, C, accumulate, L.ptr(out[:, 8:]), ld,
                                               L.ptr(inds), L.ptr(wgts), L.stream()))
    want, wi, ww = PV.np_trilinear_devoxelize(vox, grid.cpu().numpy().reshape(B, r ** 3, C), r)
    if accumulate:
        want = want + base[:, 8:8 + C].cpu().numpy().reshape(B, N, C)
    assert np.array_equal(inds.cpu().numpy(), wi)
    assert np.abs(wgts.cpu().numpy() - ww).max() <= 4e-7
    assert rel_err(out[:, 8:8 + C].reshape(B, N, C), want) < 2e-6
    assert torch.equal(out[:, :8], base[:, :8]) and torch.equal(out[:, 8 + C:], base[:, 8 + C:])


def test_trilinear_devoxelize_forward_op_in_reference_layout():
    B, N, r, C = 2, 300, 6, 16
    vox = boundary_vox(B, N, r, 9)
    feats = rnd(B, C, r, r, r, seed=9)
    outs, inds, wgts = ops.trilinear_devoxelize_forward(r, False, torch.from_numpy(vox).permute(0, 2, 1), feats.cpu())
    assert not outs.is_cuda and tuple(outs.shape) == (B, C, N) and inds.dtype == torch.int32
    want, wi, _ = PV.np_trilinear_devoxelize(vox, feats.cpu().numpy().reshape(B, C, -1).transpose(0, 2, 1), r)
    assert np.array_equal(inds.numpy(), wi) and rel_err(outs.permute(0, 2, 1), want) < 2e-6


# ------------------------------------------------------------------------------------------------------- model
@pytest.mark.parametrize("tag", ["shipped", "odd"])
def test_model_matches_recorded_reference(tag):
    sd, cfg, inp, g = PS.recorded_case(tag)
    taps = {}
    out = M.PVCNNB200(sd, cfg).forward(inp, taps=taps)
    PS.check_recorded(g, tag, out, taps, 1e-4)


@pytest.fixture(scope="module")
def shipped():
    sd, extra = H.state_dict("pvcnn_s3dis.manifest.json", 1)
    return sd, extra["cfg"], M.PVCNNB200(sd, extra["cfg"])


def test_model_matches_port_at_the_shipped_size(shipped):
    sd, cfg, net = shipped
    inp = PS.pvcnn_inputs(2, 40960, 600, cfg)
    got = net.forward(inp)
    with torch.no_grad():
        want = PV.pvcnn_forward({k: v.cuda().double() if v.is_floating_point() else v.cuda() for k, v in sd.items()},
                                {k: v.cuda().double() for k, v in inp.items()}, cfg)
    assert rel_err(got, want) <= 1e-4


def test_graphed_forward_is_the_eager_forward_and_launches_do_not_depend_on_the_cloud(shipped):
    _, cfg, net = shipped
    a, b = ({k: v.cuda() for k, v in PS.pvcnn_inputs(1, 8192, s, cfg).items()} for s in (610, 620))
    count = L.lib().o3dml_launch_count
    n0 = count()
    ea = net.forward(a).clone()
    n1 = count()
    eb = net.forward(b).clone()
    n2 = count()
    assert n1 - n0 == n2 - n1 > 0
    assert torch.equal(net.forward_graphed(a), ea) and torch.equal(net.forward_graphed(b), eb)
    assert torch.equal(net.forward_graphed(a), ea)


def test_model_refuses_what_it_does_not_build(shipped):
    sd, cfg, net = shipped
    with pytest.raises(RuntimeError, match="with_se"):
        M.PVCNNB200(sd, dict(cfg, with_se=True))
    with pytest.raises(RuntimeError, match="input channels"):
        M.PVCNNB200(sd, dict(cfg, extra_feature_channels=3))
    with pytest.raises(RuntimeError, match="channels"):
        net.forward(dict(point=torch.zeros(1, 3, 64), feat=torch.zeros(1, 4, 64)))


PATCH_SCRIPT = """
import sys
import numpy as np, torch
sys.path.insert(0, %r)
from oracle.make_ref_snapshot import ref_root
from open3d_ml_b200 import shim, pvcnn
import pvcnn_support as PS
shim.install(ref_root())
from ml3d.torch.models.pvcnn import PVCNN
sd, cfg, inp, g = PS.recorded_case("odd")
net = PVCNN(device="cuda", num_classes=cfg["num_classes"], extra_feature_channels=cfg["extra_feature_channels"],
            width_multiplier=cfg["width_multiplier"], voxel_resolution_multiplier=cfg["voxel_resolution_multiplier"])
net.load_state_dict(sd, strict=True)
net.eval()
out = pvcnn.patch_reference_model(net)(inp)
print("ERR", float(np.abs(
    out.cpu().reshape(-1)[torch.from_numpy(g["odd.logits_idx"])].numpy() - g["odd.logits"]).max() /
    np.abs(g["odd.logits"]).max()))
"""


@pytest.mark.skipif(ref_root() is None, reason="no reference tree or snapshot of it")
def test_patch_reference_model_runs_the_reference_class_on_the_fused_path():
    """In a process of its own: the shim owns sys.modules['open3d']."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here]))
    r = subprocess.run([sys.executable, "-c", PATCH_SCRIPT % here], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    err = float(r.stdout.split("ERR")[1])
    assert err <= 1e-4, err
