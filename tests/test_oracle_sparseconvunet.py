"""The SparseConvUnet oracle without a GPU: the float64 port against the logits recorded from the unmodified reference
class, and the lattice rules of DESIGN.md section 2: the parent and 2^3 cell of a voxel against the reference's own
calculate_grid and the oracle sparse convolution's cell rule, at level 0 (k + 0.5) and deeper (m + 0.25); the 3^3
table; the state_dict layout the port and the fused forward walk."""
import numpy as np
import pytest
import torch

from oracle import sparseconvunet as SP
import sparseconvunet_support as SS


@pytest.mark.parametrize("tag", SS.TAGS)
def test_port_matches_recorded_reference(tag):
    sd, cfg, batch, want = SS.recorded_case(tag)
    with torch.no_grad():
        got = SP.sparseconvunet_forward(sd, batch, cfg)
    assert tuple(got.shape) == tuple(want.shape)
    assert SS.rel_err(got, want) < 1e-5


@pytest.mark.parametrize("frac", [0.5, 0.25])
def test_parent_and_cell_match_the_reference_calculate_grid(frac):
    """The coarse lattice of the reference's calculate_grid (called itself) and, per fine voxel, the coarse voxel and
    kernel cell through which the oracle's strided and transposed 2^3 convolutions connect them (one-hot features
    through a kernel that maps cell c to column c), against floor(k / 2) and k mod 2."""
    from oracle import ops as O
    ref = SP.bind_sparseconvunet()
    rng = np.random.default_rng(7)
    k = np.unique(rng.integers(0, 30, (600, 3)), axis=0)
    pos = (k + frac).astype(np.float32)
    out = ref.calculate_grid(torch.from_numpy(pos)).numpy()
    coarse, parent, cell = SP.np_parent_cell(k)
    assert np.array_equal(out, (coarse * 2 + 0.5).astype(out.dtype))
    ident = np.eye(8, dtype=np.float32).reshape(2, 2, 2, 1, 8)
    down = O.c_sparse_conv(np.ones((len(k), 1), np.float32), pos, out, 1.0, [-0.5] * 3, ident)
    assert np.array_equal(down.sum(0), np.bincount(cell, minlength=8))        # each voxel lands in one cell
    one = np.zeros((len(coarse), 8), np.float32)
    one[parent, cell] = 1
    # the strided convolution of the fine voxel's one-hot id: coarse row parent(v) column cell(v) holds exactly v
    ids = np.arange(len(k), dtype=np.float32)[:, None] + 1
    got = O.c_sparse_conv(ids, pos, out, 1.0, [-0.5] * 3, ident)
    assert np.array_equal(got[parent, cell], ids[:, 0]) and np.count_nonzero(got) == len(k)
    # the transposed one from the coarse positions the UNet passes (2 * out / 2): fine v reads column cell(v) of parent(v)
    cf = np.arange(len(coarse), dtype=np.float32)[:, None] + 1
    up = O.c_sparse_conv(cf, (2 * (out / 2)).astype(np.float32), pos, 1.0, [-0.5] * 3, ident, transpose=True)
    assert np.array_equal(up[np.arange(len(k)), cell], parent + 1.0) and np.count_nonzero(up) == len(k)


@pytest.mark.parametrize("frac", [0.5, 0.25])
def test_parent_and_cell_match_a_restatement_of_calculate_grid(frac):
    rng = np.random.default_rng(3)
    k = np.unique(rng.integers(0, 40, (3000, 3)), axis=0)
    pos = k + frac
    coarse, parent, cell = SP.np_parent_cell(k)
    out, row, rcell = SP.np_calculate_grid_parent_cell(pos)
    assert np.array_equal(out, coarse * 2 + 0.5)           # calculate_grid's cells are the even ones, 2 m + 0.5
    assert np.array_equal(row, parent) and np.array_equal(rcell, cell)
    # the transposed convolution's cell, floor(out - in + offset + 1) with in = 2 * (m + 0.25), is the same
    tcell = np.floor(pos - 2 * (coarse[parent] + 0.25) - 0.5 + 1.0).astype(np.int64)
    assert np.array_equal((tcell[:, 0] * 2 + tcell[:, 1]) * 2 + tcell[:, 2], cell)


def test_sub_table_against_brute_force():
    rng = np.random.default_rng(4)
    k = np.unique(rng.integers(0, 12, (500, 3)), axis=0)
    t = SP.np_sub_table(k)
    where = {tuple(v): i for i, v in enumerate(k)}
    cells = [(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)]
    for i, v in enumerate(k):
        for c, d in enumerate(cells):
            assert t[i, c] == where.get((v[0] + d[0], v[1] + d[1], v[2] + d[2]), len(k))


@pytest.mark.parametrize("residual,reps", [(True, 1), (False, 2)])
def test_layout_walks_the_state_dict(residual, reps):
    from open3d_ml_b200 import sparseconvunet as M
    cfg = dict(multiplier=8, conv_block_reps=reps, residual_blocks=residual, num_classes=5)
    sd = SP.seeded_state_dict(cfg)
    lay = M.unet_layout([8 * (i + 1) for i in range(7)], residual, reps)
    used = set()
    for i, s in enumerate(lay):
        p = "unet.net.%d." % i
        keys = {k for k in sd if k.startswith(p)}
        used |= keys
        assert bool(keys) == (s[0] in ("bn", "sub", "down", "up", "res")), (i, s, keys)
    assert {k for k in sd if k.startswith("unet.")} == used


def test_port_input_layer_means_and_maps_points():
    cfg = dict(multiplier=4, conv_block_reps=1, residual_blocks=False, num_classes=3)
    sd = SP.seeded_state_dict(cfg)
    pts = np.array([[1.5, 1.5, 1.5], [1.5, 1.5, 1.5], [9.5, 3.5, 1.5]], np.float32)
    feat = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    out = SP.sparseconvunet_item(sd, cfg, pts, feat)
    assert out.shape == (3, 3) and torch.equal(out[0], out[1]) and not torch.equal(out[0], out[2])
    # the same voxel once, with the mean feature, gives the same row
    one = SP.sparseconvunet_item(sd, cfg, pts[1:], np.array([[0.5, 0.5, 0], [0, 0, 1]], np.float32))
    assert torch.allclose(one[0], out[0], rtol=1e-12, atol=1e-12)
