"""continuous_conv_transpose, invert_neighbors_list and layers.ContinuousConvTranspose on the GPU: the op against the
float64 oracle over the forward's parameter grid and at its shape and input edges, the inversion bit-equal to its
oracle and its refusal of 2^32 entries, and the layer against oracle search + inversion + transpose and as the
adjoint of the forward layer.  The launch counts and exact workspaces of both C entries are checked with every other
entry's (tests/abi_cases.py)."""
import numpy as np
import pytest
import torch

import open3d_ml_b200 as M
from open3d_ml_b200 import _lib as L, layers as LY
from oracle import ops as O
import cconv_transpose_oracle as R
from conftest import rel_err

pytestmark = pytest.mark.gpu

MAPPING = {"identity": 0, "ball_to_cube_radial": 1}
INTERP = {"nearest_neighbor": 0, "linear": 1, "linear_border": 2}
GRID = [("identity", "nearest_neighbor", True, False), ("ball_to_cube_radial", "linear", True, True),
        ("ball_to_cube_radial", "linear_border", False, False), ("identity", "linear", False, True)]


def T(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def graph(rng, n, m, ext):
    """Positions of n inputs and m outputs in the unit cube, the forward lists (outputs within ext / 2 of each input,
    from the oracle's search) and their inversion (inputs of each output)."""
    ip = rng.random((n, 3)).astype(np.float32)
    op = rng.random((m, 3)).astype(np.float32)
    fidx, fsplits, _ = O.c_radius(op, ip, ext / 2)
    tidx, tsplits, perm = R.invert_neighbors_list(m, fidx, fsplits)
    return ip, op, fidx.astype(np.int64), fsplits, tidx, tsplits, perm


def run_op(filt, op, oimp, ext, off, ip, feat, isum, fsplits, tidx, nimp, tsplits, mapping, interp, align, normalize,
           index_dtype=torch.int64, empty=torch.empty(0)):
    def opt(a):
        return empty if a is None else T(a)
    return M.ops.continuous_conv_transpose(
        T(filt), T(op), opt(oimp), torch.tensor(np.asarray(ext, np.float32).reshape(-1)), torch.tensor(off), T(ip),
        T(feat), torch.empty(0, dtype=torch.int64), opt(isum), None if fsplits is None else T(fsplits),
        T(tidx, index_dtype), opt(nimp), T(tsplits), align, mapping, normalize, interp)


def ref_op(filt, op, oimp, ext, off, ip, feat, isum, fsplits, tidx, nimp, tsplits, mapping, interp, align, normalize):
    return R.continuous_conv_transpose(filt, op, oimp, ext, off, ip, feat, isum, fsplits, tidx, nimp, tsplits, align,
                                       MAPPING[mapping], normalize, INTERP[interp])


# ------------------------------------------------------------------------------------------------------ the op
@pytest.mark.parametrize("cin,cout,n,m", [(6, 10, 200, 600), (129, 640, 40, 60)])
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("mapping,interp,align,normalize", GRID)
def test_op_vs_oracle(mapping, interp, align, normalize, index_dtype, cin, cout, n, m):
    """Cin 129 stages each input row in two passes of the 128-thread CTA and Cout 640 gives each thread 5
    accumulators; the smaller graph keeps the oracle's [entries, Cin, Cout] gathers small."""
    rng = np.random.default_rng(41)
    ext = 0.5
    ip, op, fidx, fsplits, tidx, tsplits, perm = graph(rng, n, m, ext)
    filt = rng.standard_normal((3, 4, 5, cin, cout)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    nimp = rng.random(len(tidx)).astype(np.float32)
    oimp = rng.random(m).astype(np.float32)
    isum = (rng.random(n) + 0.5).astype(np.float32)
    off = [0.1, 0.0, -0.1]
    for e in ([ext], (rng.random(n) * 0.6 + 0.2).astype(np.float32)):          # scalar and per-input extents
        for imp_sum in (isum, None):                                             # None: the forward list lengths
            args = (filt, op, oimp, e, off, ip, feat, imp_sum, fsplits, tidx, nimp, tsplits, mapping, interp, align,
                    normalize)
            got = run_op(*args, index_dtype=index_dtype)
            assert got.is_cuda and got.shape == (m, cout)
            assert rel_err(got, ref_op(*args)) < 1e-4


def test_op_edges():
    """Extent 0, empty importance tensors, outputs without neighbours, inputs without forward neighbours under
    normalize (a zero divisor scales by 1), CPU tensors in and out."""
    rng = np.random.default_rng(42)
    n, m, cin, cout = 40, 30, 5, 7
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    filt = rng.standard_normal((2, 3, 2, cin, cout)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    lens = rng.integers(0, 4, m)
    lens[::3] = 0                                                                 # outputs with no neighbours
    tsplits = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    tidx = rng.integers(0, n, tsplits[-1])
    flens = rng.integers(0, 3, n)
    flens[::2] = 0                                                                # inputs with no forward neighbours
    fsplits = np.concatenate([[0], np.cumsum(flens)]).astype(np.int64)
    for ext in ([0.0], [0.7]):
        for mapping, interp, align, normalize in GRID:
            args = (filt, op, None, ext, [0.2, 0.0, 0.1], ip, feat, None, fsplits, tidx, None, tsplits, mapping,
                    interp, align, normalize)
            got = run_op(*args)
            want = ref_op(*args)
            assert rel_err(got, want) < 1e-4
            assert bool((got[torch.from_numpy(lens == 0).cuda()] == 0).all())
    got = M.ops.continuous_conv_transpose(
        torch.from_numpy(filt), torch.from_numpy(op), torch.empty(0), torch.tensor([0.7]), torch.zeros(3),
        torch.from_numpy(ip), torch.from_numpy(feat), torch.empty(0, dtype=torch.int32), torch.empty(0),
        torch.from_numpy(fsplits), torch.from_numpy(tidx).int(), torch.empty(0), torch.from_numpy(tsplits),
        normalize=True)
    assert not got.is_cuda
    want = R.continuous_conv_transpose(filt, op, None, [0.7], [0, 0, 0], ip, feat, None, fsplits, tidx, None, tsplits,
                                       False, 1, True, 1)
    assert rel_err(got, want) < 1e-4


def test_op_empty_sides_and_widest_output():
    rng = np.random.default_rng(43)
    cin = 4
    filt = rng.standard_normal((2, 2, 2, cin, 1024)).astype(np.float32)
    m = 6
    op = rng.random((m, 3)).astype(np.float32)
    # num_inp = 0: every list is empty, the output is zero
    empty = np.zeros(m + 1, np.int64)
    got = run_op(filt, op, rng.random(m).astype(np.float32), [0.5], [0, 0, 0], np.zeros((0, 3), np.float32),
                 np.zeros((0, cin), np.float32), None, np.zeros(1, np.int64), np.zeros(0, np.int64), None, empty,
                 "ball_to_cube_radial", "linear", True, True)
    assert got.shape == (m, 1024) and bool((got == 0).all())
    # num_out = 0
    ip = rng.random((5, 3)).astype(np.float32)
    got = run_op(filt, np.zeros((0, 3), np.float32), None, [0.5], [0, 0, 0], ip,
                 rng.standard_normal((5, cin)).astype(np.float32), None, None, np.zeros(0, np.int64), None,
                 np.zeros(1, np.int64), "identity", "linear", False, False)
    assert got.shape == (0, 1024)
    # Cout = 1024: every thread of the CTA holds eight output channels
    ip, op, fidx, fsplits, tidx, tsplits, perm = graph(rng, 50, 40, 0.6)
    feat = rng.standard_normal((50, cin)).astype(np.float32)
    args = (filt, op, None, [0.6], [0, 0, 0], ip, feat, None, fsplits, tidx, None, tsplits, "ball_to_cube_radial",
            "linear", True, True)
    assert rel_err(run_op(*args), ref_op(*args)) < 1e-4


def test_non_finite_features_propagate_as_in_the_forward():
    rng = np.random.default_rng(44)
    n, m, cin, cout = 60, 80, 3, 4
    ip, op, fidx, fsplits, tidx, tsplits, perm = graph(rng, n, m, 0.6)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    feat[3, 1], feat[10, 0] = np.nan, np.inf
    filt = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    nimp = rng.random(len(tidx)).astype(np.float32)
    nimp[::5] = 0                                       # zero importance does not mask a non-finite feature
    args = (filt, op, None, [0.6], [0, 0, 0], ip, feat, None, fsplits, tidx, nimp, tsplits, "ball_to_cube_radial",
            "linear", True, False)
    got, want = run_op(*args).cpu().numpy(), ref_op(*args)
    assert np.isnan(want).any()
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
    ok = np.isfinite(want)
    assert np.abs(got[ok] - want[ok]).max() < 1e-4 * np.abs(want[ok]).max()


def test_op_refusals():
    rng = np.random.default_rng(45)
    ip, op, fidx, fsplits, tidx, tsplits, perm = graph(rng, 20, 20, 0.6)
    feat = rng.standard_normal((20, 3)).astype(np.float32)

    def call(filt=np.zeros((2, 2, 2, 3, 4), np.float32), fs=fsplits, normalize=False, mapping="identity",
             interp="linear", idx_dtype=torch.int64, ts=tsplits):
        return run_op(filt, op, None, [0.6], [0, 0, 0], ip, feat, None, fs, tidx, None, ts, mapping, interp, False,
                      normalize, index_dtype=idx_dtype)
    with pytest.raises(RuntimeError, match="normalize"):
        call(fs=None, normalize=True)
    with pytest.raises(RuntimeError, match="coordinate_mapping"):
        call(mapping="ball_to_cube_volume_preserving")
    with pytest.raises(RuntimeError, match="interpolation"):
        call(interp="cubic")
    with pytest.raises(RuntimeError, match="out_channels <= 1024"):
        call(filt=np.zeros((1, 1, 1, 3, 1025), np.float32))
    with pytest.raises(RuntimeError, match="12288"):
        run_op(np.zeros((1, 1, 1, 12289, 1), np.float32), op, None, [0.6], [0, 0, 0], ip,
               np.zeros((20, 12289), np.float32), None, None, tidx, None, tsplits, "identity", "linear", False, False)
    with pytest.raises(RuntimeError, match="filters"):
        call(filt=np.zeros((2, 2, 3, 4), np.float32))
    with pytest.raises(RuntimeError, match="int32 or int64"):
        call(idx_dtype=torch.int16)
    with pytest.raises(RuntimeError, match="row_splits"):
        call(ts=tsplits[:-1])
    with pytest.raises(RuntimeError, match=r"inp_positions must have shape \[N, 3\]"):
        run_op(np.zeros((2, 2, 2, 3, 4), np.float32), op, None, [0.6], [0, 0, 0], np.ascontiguousarray(ip[:, :2]),
               feat, None, fsplits, tidx, None, tsplits, "identity", "linear", False, False)


# ------------------------------------------------------------------------------------------- invert_neighbors_list
def lists(rng, rows, num_points, max_len, bad):
    lens = rng.integers(0, max_len + 1, rows)
    splits = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(0, max(num_points, 1), splits[-1])
    drop = rng.random(len(idx)) < bad
    idx[drop] = np.where(rng.random(drop.sum()) < 0.5, -1, num_points + rng.integers(0, 5, drop.sum()))
    return idx, splits


@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("num_points,rows,max_len,bad", [(1000, 700, 12, 0.0), (100, 3000, 9, 0.05),
                                                         (5, 2000, 6, 0.3), (500, 0, 1, 0.0), (500, 40, 0, 0.0),
                                                         (0, 30, 4, 0.0)])
def test_invert_neighbors_list_bit_equal_to_oracle(index_dtype, num_points, rows, max_len, bad):
    rng = np.random.default_rng(num_points + 7 * rows)
    idx, splits = lists(rng, rows, num_points, max_len, bad)
    ref_idx, ref_rs, perm = R.invert_neighbors_list(num_points, idx, splits)
    e = len(idx)
    attrs = [torch.empty(0), T(rng.random(e).astype(np.float32)), T(rng.standard_normal((e, 3))),
             T(rng.integers(-9, 9, e).astype(np.int32)), T(rng.integers(-9, 9, (e, 3)))]
    for a in attrs:
        r = M.ops.invert_neighbors_list(num_points, T(idx, index_dtype), T(splits), a)
        assert r.neighbors_index.dtype == index_dtype and r.neighbors_row_splits.dtype == torch.int64
        assert np.array_equal(r.neighbors_index.cpu().numpy(), ref_idx)
        assert np.array_equal(r.neighbors_row_splits.cpu().numpy(), ref_rs)
        if a.numel():
            assert r.neighbors_attributes.dtype == a.dtype
            assert np.array_equal(r.neighbors_attributes.cpu().numpy(), a.cpu().numpy()[perm])
        else:
            assert r.neighbors_attributes.numel() == 0
    kept = int(((idx >= 0) & (idx < num_points)).sum())
    assert int(ref_rs[-1]) == kept
    cpu = M.ops.invert_neighbors_list(num_points, torch.from_numpy(idx), torch.from_numpy(splits), torch.empty(0))
    assert not cpu.neighbors_index.is_cuda and np.array_equal(cpu.neighbors_index.numpy(), ref_idx)


def test_invert_neighbors_list_duplicates_in_input_order():
    idx = np.array([3, 1, 3, 3, 0, 9, 1, -2, 3], np.int64)
    splits = np.array([0, 4, 4, 7, 9], np.int64)
    r = M.ops.invert_neighbors_list(4, T(idx), T(splits), T(np.arange(9, dtype=np.float32)))
    assert r.neighbors_row_splits.tolist() == [0, 1, 3, 3, 7]
    assert r.neighbors_index.tolist() == [2, 0, 2, 0, 0, 0, 3, 2, 3]
    assert r.neighbors_attributes.tolist() == [4, 1, 6, 0, 2, 3, 8, 5, 7]


# ------------------------------------------------------------------------------------------------------ the layer
@pytest.mark.parametrize("mapping,interp,align,normalize", GRID)
def test_layer_vs_oracle_search_inversion_and_transpose(mapping, interp, align, normalize):
    rng = np.random.default_rng(46)
    n, m, cin, cout, ext = 300, 500, 6, 10, 0.5
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    oimp = rng.random(m).astype(np.float32)
    with torch.no_grad():
        layer = LY.ContinuousConvTranspose(cin, cout, [3, 4, 5], align_corners=align, coordinate_mapping=mapping,
                                           interpolation=interp, normalize=normalize, offset=[0.1, 0, -0.1]).eval()
        layer.bias.normal_()
        got = layer(torch.from_numpy(feat), torch.from_numpy(ip), torch.from_numpy(op), ext,
                    out_importance=torch.from_numpy(oimp))
        assert not got.is_cuda                            # CPU in, CPU out
        got_cuda = layer(T(feat), T(ip), T(op), torch.tensor([ext]), out_importance=T(oimp))
        assert got_cuda.is_cuda and torch.equal(got_cuda.cpu(), got)
    fidx, fsplits, _ = O.c_radius(op, ip, ext / 2)
    tidx, tsplits, _ = R.invert_neighbors_list(m, fidx, fsplits)
    want = R.continuous_conv_transpose(layer.kernel.detach().numpy(), op, oimp, [ext], [0.1, 0, -0.1], ip, feat, None,
                                       fsplits, tidx, None, tsplits, align, MAPPING[mapping], normalize, INTERP[interp])
    assert rel_err(got, want + layer.bias.detach().numpy()) < 1e-4


@pytest.mark.parametrize("normalize", [False, True])
def test_layer_is_the_adjoint_of_the_forward_layer(normalize):
    """<F(y), x> = <y, T(x)> for the forward layer F with the kernel's channel axes swapped (no bias)."""
    rng = np.random.default_rng(47)
    n, m, cin, cout, ext = 400, 900, 8, 5, 0.35
    ip, op = T(rng.random((n, 3)).astype(np.float32)), T(rng.random((m, 3)).astype(np.float32))
    x, y = T(rng.standard_normal((n, cin)).astype(np.float32)), T(rng.standard_normal((m, cout)).astype(np.float32))
    kw = dict(align_corners=True, coordinate_mapping="ball_to_cube_radial", interpolation="linear",
              normalize=normalize, use_bias=False)
    with torch.no_grad():
        t = LY.ContinuousConvTranspose(cin, cout, [4, 4, 4], **kw).eval()
        f = LY.ContinuousConv(cout, cin, [4, 4, 4], **kw).eval()
        f.kernel.copy_(t.kernel.transpose(-1, -2))
        tx = t(x, ip, op, ext)
        fy = f(y, op, ip, ext)
    a, b = (fy.double() * x.double()).sum(), (y.double() * tx.double()).sum()
    terms = (fy.double() * x.double()).abs().sum() + (y.double() * tx.double()).abs().sum()
    assert float(terms) > 0 and float((a - b).abs()) <= 1e-4 * float(terms)       # fp32 sums on both sides


def test_layer_refusals_and_state_dict():
    cc = LY.ContinuousConv(3, 4, [3, 3, 3], offset=[0.1, 0.2, 0.3])
    t = LY.ContinuousConvTranspose(3, 4, [3, 3, 3])
    t.load_state_dict(cc.state_dict())                   # same parameter and buffer names
    assert torch.equal(t.kernel, cc.kernel) and torch.equal(t.offset, cc.offset)
    x, p = torch.rand(10, 3), torch.rand(10, 3)
    with pytest.raises(RuntimeError, match="one extent"):
        t(x, p, p, torch.full((10,), 0.3))
    for k in ("user_neighbors_index", "user_neighbors_row_splits", "user_neighbors_importance"):
        with pytest.raises(RuntimeError, match=k):
            t(x, p, p, 0.3, **{k: torch.zeros(1, dtype=torch.int32)})
    with pytest.raises(RuntimeError, match="window_function"):
        LY.ContinuousConvTranspose(3, 4, [3, 3, 3], window_function=lambda r: 1 - r)
    with pytest.raises(RuntimeError, match="use_dense_layer_for_center"):
        LY.ContinuousConvTranspose(3, 4, [3, 3, 3], use_dense_layer_for_center=True)


# --------------------------------------------------------------------------------------------------- the C ABI
def test_invert_refuses_2_to_the_32_entries():
    rs = torch.zeros(2, dtype=torch.int64).cuda()
    out_rs = torch.empty(11, dtype=torch.int64).cuda()
    assert L.lib().o3dml_invert_neighbors_list(10, None, 1, L.ptr(rs), 1, 1 << 32, None, L.ptr(out_rs), None, None, 0,
                                               L.stream()) == 1
    assert "2^32" in L.lib().o3dml_last_error().decode()
