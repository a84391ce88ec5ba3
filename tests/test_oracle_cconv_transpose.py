"""The float64 oracle of continuous_conv_transpose and invert_neighbors_list, pinned without a GPU: the transposed op
is the exact adjoint of continuous_conv's oracle, known answers on a lattice and for a constant filter, and the
inversion against a numpy stable-argsort restatement.  The shim resolves the new names without touching CUDA."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ops as O
import cconv_transpose_oracle as R
from cconv_cases import FAR
from conftest import ROOT


def np_invert(num_points, idx, splits):
    """invert_neighbors_list restated: a stable argsort of the entries by id, out-of-range ids keyed past the end."""
    idx, splits = np.asarray(idx, np.int64), np.asarray(splits, np.int64)
    row = np.repeat(np.arange(len(splits) - 1), np.diff(splits))
    key = np.where((idx >= 0) & (idx < num_points), idx, num_points)
    perm = np.argsort(key, kind="stable")
    rs = np.searchsorted(key[perm], np.arange(num_points + 1), side="left")
    return row[perm], rs.astype(np.int64), perm


def random_lists(rng, rows, num_points, max_len, bad=0.0):
    lens = rng.integers(0, max_len + 1, rows)
    splits = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(0, num_points, splits[-1]) if num_points else np.zeros(splits[-1], np.int64)
    if bad:
        drop = rng.random(len(idx)) < bad
        idx[drop] = np.where(rng.random(drop.sum()) < 0.5, -1 - rng.integers(0, 3, drop.sum()),
                             num_points + rng.integers(0, 3, drop.sum()))
    return idx, splits


def adjoint_gap(rng, mapping, interp, align, normalize, importances, per_point, by_count=False, far=False):
    """(|<z, x> - <y, T(x)>|, sum of |terms|) for one random mirrored pair of graphs.  far: the first 18 outputs are
    moved 1e3, 1e9 and 1e12 out on either side of each axis, so their entries take a border cell or weigh 0."""
    num_inp, num_out, cin, cout = 30, 50, 3, 4
    inp_pos = rng.random((num_inp, 3)).astype(np.float32)
    out_pos = rng.random((num_out, 3)).astype(np.float32)
    if far:
        for k, (a, side, mag) in enumerate(itertools.product(range(3), (-1, 1), FAR)):
            out_pos[k, a] += np.float32(side * mag)
    W = rng.standard_normal((3, 4, 2, cin, cout)).astype(np.float32)
    G = np.ascontiguousarray(W.transpose(0, 1, 2, 4, 3))
    x = rng.standard_normal((num_inp, cin)).astype(np.float32)
    y = rng.standard_normal((num_out, cout)).astype(np.float32)
    ext = (rng.random(num_inp) * 0.8 + 0.4).astype(np.float32) if per_point else np.float32([0.9])
    off = [0.1, -0.05, 0.0]
    fwd_idx, fwd_splits = random_lists(rng, num_inp, num_out, 6)      # input i -> outputs j (with duplicates)
    nimp = (rng.random(len(fwd_idx)) + 0.2).astype(np.float32) if importances else None
    oimp = (rng.random(num_out) + 0.2).astype(np.float32) if importances else None
    z = O.c_continuous_conv(G, inp_pos, ext, off, out_pos, y, oimp, fwd_idx, nimp, fwd_splits, align, mapping,
                            normalize, interp)
    t_idx, t_splits, perm = R.invert_neighbors_list(num_out, fwd_idx, fwd_splits)
    imp_sum = None
    if not by_count:
        w = (np.ones(len(fwd_idx)) if nimp is None else nimp.astype(np.float64)) * \
            (1.0 if oimp is None else oimp[fwd_idx].astype(np.float64))
        imp_sum = np.array([w[a:b].sum() for a, b in zip(fwd_splits[:-1], fwd_splits[1:])], np.float32)
    T = R.continuous_conv_transpose(W, out_pos, oimp, ext, off, inp_pos, x, imp_sum, fwd_splits, t_idx,
                                    None if nimp is None else nimp[perm], t_splits, align, mapping, normalize, interp)
    a = (z.astype(np.float64) * x).sum()
    b = (y.astype(np.float64) * T).sum()
    terms = np.abs(z.astype(np.float64) * x).sum() + np.abs(y.astype(np.float64) * T).sum()
    return abs(a - b), terms


@pytest.mark.parametrize("interp", [0, 1, 2])
@pytest.mark.parametrize("mapping", [0, 1])
@pytest.mark.parametrize("align", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
def test_transpose_oracle_is_the_adjoint_of_the_forward(interp, mapping, align, normalize):
    rng = np.random.default_rng(100 + 12 * interp + 4 * mapping + 2 * align + normalize)
    for importances, per_point, far in ((False, False, False), (True, False, False), (True, True, False),
                                        (True, True, True)):
        gap, terms = adjoint_gap(rng, mapping, interp, align, normalize, importances, per_point, far=far)
        assert terms > 0 and gap <= 1e-5 * terms, (importances, per_point, far, gap, terms)


def test_adjoint_with_the_neighbour_count_as_normaliser():
    """Without importances the forward normalises by the list length, which is what the transposed op reads from
    inp_neighbors_row_splits when no importance sum is given."""
    rng = np.random.default_rng(7)
    for interp in (0, 1, 2):
        gap, terms = adjoint_gap(rng, 1, interp, True, True, False, True, by_count=True)
        assert gap <= 1e-5 * terms, (interp, gap, terms)


def test_one_hot_filter_on_a_lattice_selects_the_cell():
    """Nearest interpolation, identity mapping, align_corners, extent 2h: an output at lattice offset d from the input
    lands in cell d + 1, so a filter that is one-hot per cell returns that cell's id."""
    h = 0.25
    d = np.stack(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1], indexing="ij"), -1).reshape(-1, 3)
    centre = np.float32([[0.3, 0.4, 0.5]])
    out_pos = (centre + d * h).astype(np.float32)
    filt = np.zeros((3, 3, 3, 1, 27), np.float32)
    for z in range(3):
        for y in range(3):
            for x in range(3):
                filt[z, y, x, 0, (z * 3 + y) * 3 + x] = 1
    idx = np.zeros(27, np.int64)                      # every output has the one input as neighbour
    splits = np.arange(28, dtype=np.int64)
    got = R.continuous_conv_transpose(filt, out_pos, None, [2 * h], [0, 0, 0], centre, np.float32([[1.0]]), None,
                                      None, idx, None, splits, True, 0, False, 0)
    cell = ((d[:, 2] + 1) * 3 + (d[:, 1] + 1)) * 3 + (d[:, 0] + 1)
    assert np.array_equal(got, np.eye(27, dtype=np.float32)[cell])


@pytest.mark.parametrize("mapping,interp", [(0, 0), (1, 1), (1, 2)])
def test_constant_filter_gives_importance_weighted_sums(mapping, interp):
    rng = np.random.default_rng(3)
    num_inp, num_out, cin, cout = 20, 15, 3, 5
    inp_pos = rng.random((num_inp, 3)).astype(np.float32)
    out_pos = rng.random((num_out, 3)).astype(np.float32)
    x = rng.standard_normal((num_inp, cin)).astype(np.float32)
    Wc = rng.standard_normal((cin, cout)).astype(np.float32)
    filt = np.broadcast_to(Wc, (2, 2, 2, cin, cout)).copy()
    idx, splits = random_lists(rng, num_out, num_inp, 5)
    nimp = rng.random(len(idx)).astype(np.float32)
    oimp = rng.random(num_out).astype(np.float32)
    isum = (rng.random(num_inp) + 0.5).astype(np.float32)
    isum[0] = 0                                        # a zero divisor scales by 1
    # linear_border zeroes corners outside the filter: keep every point well inside (extent 8 -> |p| <= 0.25)
    got = R.continuous_conv_transpose(filt, out_pos, oimp, [8.0], [0, 0, 0], inp_pos, x, isum, None, idx, nimp,
                                      splits, True, mapping, True, interp)
    s = np.where(isum != 0, 1.0 / np.where(isum != 0, isum, 1), 1.0)
    want = np.stack([oimp[j] * sum(nimp[e] * s[idx[e]] * x[idx[e]].astype(np.float64) for e in range(a, b)) @ Wc
                     if b > a else np.zeros(cout) for j, (a, b) in enumerate(zip(splits[:-1], splits[1:]))])
    assert np.abs(got - want).max() < 1e-5 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("num_points,rows,max_len,bad", [(50, 40, 8, 0.0), (50, 40, 8, 0.2), (7, 100, 12, 0.1),
                                                         (30, 0, 4, 0.0), (30, 20, 0, 0.0), (0, 10, 3, 0.0),
                                                         (5, 10, 4, 1.0)])
def test_inversion_oracle_equals_a_stable_argsort(num_points, rows, max_len, bad):
    rng = np.random.default_rng(num_points * 131 + rows)
    idx, splits = random_lists(rng, rows, num_points, max_len, bad)
    if num_points == 0:
        idx[:] = rng.integers(-2, 3, len(idx))        # everything is out of range
    got = R.invert_neighbors_list(num_points, idx, splits)
    want = np_invert(num_points, idx, splits)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    kept = ((idx >= 0) & (idx < num_points)).sum()
    assert got[1][-1] == kept and got[1][0] == 0
    assert np.array_equal(idx[got[2][kept:]], idx[~((idx >= 0) & (idx < num_points))])    # dropped, in input order


def test_shim_resolves_the_transposed_names_without_cuda():
    code = ("import torch, open3d_ml_b200.shim as shim\n"
            "shim.install()\n"
            "from open3d.ml.torch.ops import continuous_conv_transpose, invert_neighbors_list\n"
            "from open3d.ml.torch.layers import ContinuousConvTranspose\n"
            "from open3d_ml_b200 import _lib, layers, ops\n"
            "assert continuous_conv_transpose is ops.continuous_conv_transpose\n"
            "assert invert_neighbors_list is ops.invert_neighbors_list\n"
            "assert ContinuousConvTranspose is layers.ContinuousConvTranspose\n"
            "assert _lib._lib is None and not torch.cuda.is_initialized()\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
