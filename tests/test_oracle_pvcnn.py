"""The PVCNN oracle without a GPU: the torch port against the logits and taps recorded from the unmodified reference
class, and the float64 voxel and devoxelization rules of DESIGN.md section 2 on constructed cases."""
import numpy as np
import pytest
import torch

from oracle import pvcnn as PV
import pvcnn_support as PS


@pytest.mark.parametrize("tag", ["shipped", "odd"])
def test_port_matches_recorded_reference(tag):
    sd, cfg, inp, g = PS.recorded_case(tag)
    taps = {}
    with torch.no_grad():
        out = PV.pvcnn_forward(sd, inp, cfg, taps=taps)
    assert tuple(out.shape) == tuple(g[tag + ".logits_shape"])
    PS.check_recorded(g, tag, out, taps, 1e-5)


def test_exact_halves_round_to_even_and_clamp():
    v, cell = PV.np_pv_voxel_cells(PS.tie_cloud(), PS.TIE_R, eps=0.0)
    assert np.array_equal(v[0, :, 0], PS.TIE_VOX_X) and np.all(v[0, :, 1:] == 2.0)
    assert np.array_equal(cell[0], PS.tie_cells())
    # the torch port rounds the same way
    q = torch.round(PV.pv_voxel_coords(torch.from_numpy(PS.tie_cloud()).permute(0, 2, 1), PS.TIE_R, eps=0.0))
    assert np.array_equal(q[0, 0].numpy(), PS.TIE_CELL_X)


@pytest.mark.parametrize("n", [1, 7])
def test_cloud_of_identical_points_lands_in_the_centre(n):
    """Largest norm 0: eps alone is the denominator, every coordinate is r / 2, and 2.5 rounds to 2."""
    pts = np.full((2, n, 3), 3.25, np.float32)
    v, cell = PV.np_pv_voxel_cells(pts, 5)
    assert np.all(v == 2.5)
    assert np.array_equal(cell, np.array([[62] * n, [125 + 62] * n]))
    grid = PV.np_avg_voxelize(np.ones((2, n, 3)), cell, 250)
    assert grid[62].tolist() == [1, 1, 1] and grid[187].tolist() == [1, 1, 1] and grid.sum() == 6


def test_avg_voxelize_is_a_mean_with_zero_for_empty_cells():
    cell = np.array([[0, 3, 3, 3]])
    grid = PV.np_avg_voxelize(np.array([[[1.0], [2.0], [4.0], [9.0]]]), cell, 8)
    assert grid[:, 0].tolist() == [1, 0, 0, 5, 0, 0, 0, 0]


def test_devoxelize_on_integer_coordinates_reads_one_cell():
    r = 4
    rng = np.random.default_rng(0)
    grid = rng.standard_normal((1, r ** 3, 3))
    vox = np.array([[[0, 0, 0], [3, 3, 3], [1, 2, 3], [3, 0, 2]]], np.float64)
    outs, inds, wgts = PV.np_trilinear_devoxelize(vox, grid, r)
    cells = ((vox[0, :, 0] * r + vox[0, :, 1]) * r + vox[0, :, 2]).astype(int)
    assert np.array_equal(outs[0], grid[0, cells])
    assert np.all(inds[0] == cells[None, :]) and inds.max() < r ** 3       # x = r - 1 never reads cell r
    assert np.all(wgts[0, 0] == 1) and np.all(wgts[0, 1:] == 0)


def test_devoxelize_weights_and_port_agree():
    r = 5
    rng = np.random.default_rng(1)
    vox = rng.uniform(0, r - 1, (2, 50, 3))
    vox[0, :5] = [[0.5, 0, 4], [4, 4, 4], [3.999, 0.001, 2], [0, 0, 0], [2, 2.5, 2]]
    grid = rng.standard_normal((2, r ** 3, 4))
    outs, inds, wgts = PV.np_trilinear_devoxelize(vox, grid, r)
    assert np.allclose(wgts.sum(1), 1, atol=1e-12) and inds.min() >= 0 and inds.max() < r ** 3
    po, pi, pw = PV.pv_trilinear_devoxelize(r, False, torch.from_numpy(vox).permute(0, 2, 1),
                                            torch.from_numpy(grid).permute(0, 2, 1).reshape(2, 4, r, r, r))
    assert np.array_equal(pi.numpy(), inds)
    assert np.allclose(pw.numpy(), wgts, atol=1e-14) and np.allclose(po.permute(0, 2, 1).numpy(), outs, atol=1e-13)


def test_margin_nudge_keeps_points_off_the_rounding_boundaries():
    pts, _ = PS.filtered_cloud(2000, 3, [24, 48])
    for r in (24, 48):
        v, _ = PV.np_pv_voxel_cells(pts[None], r)
        assert np.abs(np.abs(v - np.floor(v)) - 0.5).min() >= 1e-3
