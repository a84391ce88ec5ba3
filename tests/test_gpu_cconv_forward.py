"""continuous_conv and layers.ContinuousConv on the GPU against the float64 C oracle (oracle/ops_ref.c, which
tests/test_oracle_cconv_transpose.py holds to the independent transpose oracle): the op over the mapping /
interpolation grid, both index widths, scalar and per-output extents and every importance combination; channel
counts at the edges of the 128-thread CTA (a second pass to stage the neighbour row, 2 to 8 accumulators per thread);
filter coordinates exactly on cells, on nearest-neighbour ties and on the last cell; empty lists and sizes, extent 0
and zero normalisers; neighbours up to 1e12 extents away; non-finite features and positions; and the refusals.
The transposed instance of the same kernel is tested in tests/test_gpu_cconv_transpose.py."""
import numpy as np
import pytest
import torch

import open3d_ml_b200 as M
from open3d_ml_b200 import layers as LY
from oracle import ops as O
from cconv_cases import far_neighbours
from conftest import rel_err

pytestmark = pytest.mark.gpu

MAPPING = {"identity": 0, "ball_to_cube_radial": 1}
INTERP = {"nearest_neighbor": 0, "linear": 1, "linear_border": 2}
GRID = [("identity", "nearest_neighbor", True, False), ("ball_to_cube_radial", "linear", True, True),
        ("ball_to_cube_radial", "linear_border", False, False), ("identity", "linear", False, True)]


def T(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def run_op(filt, op, ext, off, ip, feat, iimp, idx, nimp, rs, mapping, interp, align, normalize,
           index_dtype=torch.int64, empty=torch.empty(0)):
    def opt(a):
        return empty if a is None else T(a)
    return M.ops.continuous_conv(T(filt), T(op), torch.tensor(np.asarray(ext, np.float32).reshape(-1)),
                                 torch.tensor(np.asarray(off, np.float32)), T(ip), T(feat), opt(iimp),
                                 T(idx, index_dtype), opt(nimp), T(rs), align, mapping, normalize, interp)


def ref_op(filt, op, ext, off, ip, feat, iimp, idx, nimp, rs, mapping, interp, align, normalize):
    return O.c_continuous_conv(filt, op, ext, off, ip, feat, iimp, idx, nimp, rs, align, MAPPING[mapping], normalize,
                               INTERP[interp])


def random_lists(rng, m, n, max_len):
    lens = rng.integers(0, max_len + 1, m)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return rng.integers(0, n, rs[-1]).astype(np.int64), rs


# ------------------------------------------------------------------------------------------------------ the op
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("mapping,interp,align,normalize", GRID)
def test_op_vs_oracle(mapping, interp, align, normalize, index_dtype):
    rng = np.random.default_rng(21)
    n, m, cin, cout, ext = 600, 200, 6, 10, 0.5
    ip = rng.random((n, 3)).astype(np.float32)
    op = rng.random((m, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    filt = rng.standard_normal((3, 4, 5, cin, cout)).astype(np.float32)
    idx, rs, _ = O.c_radius(ip, op, ext / 2)
    iimp = rng.random(n).astype(np.float32)
    nimp = rng.random(len(idx)).astype(np.float32)
    off = [0.1, 0.0, -0.1]
    for e in ([ext], (rng.random(m) * 0.6 + 0.2).astype(np.float32)):           # scalar and per-output extents
        for ii, ni in ((None, None), (iimp, None), (None, nimp), (iimp, nimp)):
            args = (filt, op, e, off, ip, feat, ii, idx, ni, rs, mapping, interp, align, normalize)
            got = run_op(*args, index_dtype=index_dtype)
            assert got.is_cuda and got.shape == (m, cout)
            assert rel_err(got, ref_op(*args)) < 1e-4, (len(e), ii is not None, ni is not None)


@pytest.mark.parametrize("cin,cout", [(1, 1), (129, 7), (300, 33), (5, 129), (7, 640), (3, 1024), (12288, 2)])
def test_channel_edges(cin, cout):
    """Cin > 128 stages the neighbour row in more than one pass of the CTA; Cout > 128 gives each thread 2 to 8
    accumulators.  Lists of up to 4 neighbours keep the fp32 sums short at Cin = 12288."""
    rng = np.random.default_rng(cin * 7 + cout)
    n, m = 50, 40
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    filt = rng.standard_normal((2, 3, 2, cin, cout)).astype(np.float32)
    idx, rs = random_lists(rng, m, n, 4)
    iimp = rng.random(n).astype(np.float32)
    nimp = rng.random(len(idx)).astype(np.float32)
    for mapping, interp, align, normalize in GRID:
        args = (filt, op, [1.2], [0.0, 0.1, 0.0], ip, feat, iimp, idx, nimp, rs, mapping, interp, align, normalize)
        got = run_op(*args)
        assert got.shape == (m, cout)
        assert rel_err(got, ref_op(*args)) < 1e-4, (mapping, interp)


# ---------------------------------------------------------------------------------------- exact lattice coordinates
def lattice_case(rng, radial, m=3000):
    """One neighbour per output; positions are multiples of 1/16 in [0, 1] and extents 0.5, 1 or 2, so with offsets
    in {0, +-0.25} every filter coordinate u is exact in float32 as in float64.  radial: each input sits on its
    output or is displaced along one axis, where ball_to_cube_radial is the identity (|p|_2 = |p|_inf)."""
    op = rng.integers(0, 17, (m, 3)) / 16.0
    ip = rng.integers(0, 17, (m, 3)) / 16.0
    if radial:
        axis = rng.integers(0, 4, m)                                   # 3: the input on its output (p = 0)
        ip = np.where(np.arange(3)[None, :] == axis[:, None], ip, op)
    ext = rng.choice([0.5, 1.0, 2.0], m)
    return op.astype(np.float32), ip.astype(np.float32), ext.astype(np.float32)


def filter_coords(op, ip, ext, off, sizes, align):
    S = np.array(sizes, np.float64)
    p = (ip.astype(np.float64) - op) * (2.0 / ext.astype(np.float64))[:, None] + np.asarray(off, np.float64)
    return (p + 1) * 0.5 * (S - 1) if align else (p + 1) * 0.5 * S - 0.5


@pytest.mark.parametrize("interp", ["nearest_neighbor", "linear", "linear_border"])
@pytest.mark.parametrize("align", [False, True])
@pytest.mark.parametrize("sizes", [(1, 2, 5), (3, 4, 1), (5, 3, 2)])
def test_exact_lattice_coordinates(sizes, align, interp):
    """Small-integer filters and features and dyadic weights make every result exact in float32: the kernel must
    equal the oracle bit for bit, so a cell picked one off (a tie rounded down, the last cell of linear dropped) shows.
    The cases are checked to land on nearest-neighbour ties k + 0.5, on interior cells, on the last cell S - 1 and
    outside the filter on both sides."""
    rng = np.random.default_rng(sum(sizes) * 10 + 2 * align + INTERP[interp])
    cin, cout = 3, 4
    filt = rng.integers(-4, 5, (sizes[2], sizes[1], sizes[0], cin, cout)).astype(np.float32)
    seen = {"tie": 0, "cell": 0, "last": 0, "below": 0, "above": 0}
    for mapping, offsets in (("identity", ([0, 0, 0], [0.25, -0.25, 0.0], [-0.25, 0.0, 0.25])),
                             ("ball_to_cube_radial", ([0, 0, 0],))):
        op, ip, ext = lattice_case(rng, mapping != "identity")
        m = len(op)
        feat = rng.integers(-2, 3, (m, cin)).astype(np.float32)
        idx, rs = np.arange(m, dtype=np.int64), np.arange(m + 1, dtype=np.int64)
        for off in offsets:
            args = (filt, op, ext, off, ip, feat, None, idx, None, rs, mapping, interp, align, False)
            got = run_op(*args).cpu().numpy()
            want = ref_op(*args)
            assert np.array_equal(got, want), (mapping, off, np.abs(got - want).max())
            u = filter_coords(op, ip, ext, off, sizes, align)
            for a, s in enumerate(sizes):
                if s == 1:
                    continue
                ua = u[:, a]
                seen["tie"] += int(((ua - 0.5 == np.floor(ua - 0.5)) & (ua > 0) & (ua < s - 1)).sum())
                seen["cell"] += int(((ua == np.floor(ua)) & (ua >= 0) & (ua < s - 1)).sum())
                seen["last"] += int((ua == s - 1).sum())
                seen["below"] += int((ua < -1).sum())
                seen["above"] += int((ua > s).sum())
    assert min(seen.values()) > 0, seen


# -------------------------------------------------------------------------------------------------- degenerate inputs
def test_degenerate_inputs():
    """Empty lists give exact zeros; num_out = 0 and num_inp = 0; extent 0 (every neighbour maps to `offset`) and
    per-output extents that contain 0; normalize over rows whose importances are all 0 or sum to 0 (a zero divisor
    scales by 1); duplicate neighbours in one list; CPU tensors in and out."""
    rng = np.random.default_rng(22)
    n, m, cin, cout = 40, 30, 5, 7
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    filt = rng.standard_normal((3, 2, 4, cin, cout)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    lens = rng.integers(1, 5, m)
    lens[::4] = 0                                                                  # outputs with no neighbours
    lens[1], lens[2] = 3, 4
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(0, n, rs[-1]).astype(np.int64)
    idx[rs[1]:rs[1] + 2] = idx[rs[1]]                                             # a neighbour listed twice
    nimp = rng.random(len(idx)).astype(np.float32)
    nimp[rs[1]:rs[2]] = 0                                                         # importances all 0
    nimp[rs[2]:rs[3]] = [0.5, -0.5, 0, 0]                                         # importances that sum to 0
    empty = torch.from_numpy(lens == 0).cuda()
    per_out = (rng.random(m) * 0.8 + 0.2).astype(np.float32)
    per_out[::3] = 0
    off = [0.2, 0.0, -0.3]
    for ext in ([0.0], [0.7], per_out):
        for mapping, interp, align, normalize in GRID:
            for ni in (None, nimp):
                args = (filt, op, ext, off, ip, feat, None, idx, ni, rs, mapping, interp, align, normalize)
                got = run_op(*args)
                want = ref_op(*args)
                assert rel_err(got, want) < 1e-4, (len(ext), mapping, interp, ni is not None)
                assert bool((got[empty] == 0).all())
    want = ref_op(filt, op, [0.7], off, ip, feat, None, idx, nimp, rs, "identity", "linear", False, True)
    assert np.abs(want[2]).max() > 0                                              # scaled by 1, not divided by 0
    # num_inp = 0: every list is empty and the output is zero
    got = run_op(filt, op, [0.5], off, np.zeros((0, 3), np.float32), np.zeros((0, cin), np.float32),
                 None, np.zeros(0, np.int64), None, np.zeros(m + 1, np.int64), "ball_to_cube_radial", "linear", True,
                 True)
    assert got.shape == (m, cout) and bool((got == 0).all())
    # num_out = 0
    got = run_op(filt, np.zeros((0, 3), np.float32), [0.5], off, ip, feat, rng.random(n).astype(np.float32),
                 np.zeros(0, np.int64), None, np.zeros(1, np.int64), "identity", "nearest_neighbor", True, False)
    assert got.shape == (0, cout)
    # CPU tensors in, CPU tensors out
    got = M.ops.continuous_conv(torch.from_numpy(filt), torch.from_numpy(op), torch.tensor([0.7]), torch.tensor(off),
                                torch.from_numpy(ip), torch.from_numpy(feat), torch.empty(0),
                                torch.from_numpy(idx).int(), torch.from_numpy(nimp), torch.from_numpy(rs),
                                normalize=True)
    assert not got.is_cuda
    want = O.c_continuous_conv(filt, op, [0.7], off, ip, feat, None, idx, nimp, rs, False, 1, True, 1)
    assert rel_err(got, want) < 1e-4


# ----------------------------------------------------------------------------------------------------- far neighbours
@pytest.mark.parametrize("align", [False, True])
@pytest.mark.parametrize("interp", ["nearest_neighbor", "linear", "linear_border"])
@pytest.mark.parametrize("sizes", [(3, 4, 5), (5, 1, 2)])
def test_far_neighbours_take_the_border_cell(sizes, interp, align):
    """Neighbours 1e3, 1e9 and 1e12 extents out on either side of each axis, through the op and through the layer's
    user lists: the border cell on that side (nearest, linear) or weight 0 (linear_border), as the closed form of a
    filter that holds each cell's flat index says, and as the oracle computes."""
    c = far_neighbours(sizes, align, INTERP[interp])
    for mapping in MAPPING:
        args = (c.filters, c.out_pos, [1.0], [0, 0, 0], c.inp_pos, c.feat, None, c.index, None, c.splits, mapping,
                interp, align, False)
        got = run_op(*args).cpu().numpy()
        assert np.array_equal(got, c.want), (mapping, got.ravel(), c.want.ravel())
        assert np.array_equal(ref_op(*args), c.want)
        with torch.no_grad():
            layer = LY.ContinuousConv(1, 1, list(c.filters.shape[:3]), align_corners=align, coordinate_mapping=mapping,
                                      interpolation=interp, normalize=False, use_bias=False).eval()
            layer.kernel.copy_(torch.from_numpy(c.filters))
            out = layer(T(c.feat), T(c.inp_pos), T(c.out_pos), 1.0, user_neighbors_index=T(c.index),
                        user_neighbors_row_splits=T(c.splits))
        assert np.array_equal(out.cpu().numpy(), c.want), mapping


# ------------------------------------------------------------------------------------------------------ non-finite
@pytest.mark.parametrize("mapping,interp,align,normalize", GRID)
def test_non_finite_features_and_positions_propagate_as_in_the_oracle(mapping, interp, align, normalize):
    """NaN and inf features reach every output that reads them with a nonzero interpolation weight, also at zero
    importance; a NaN or inf position takes the oracle's cells and weights (NaN weights under linear, weight 0
    under linear_border, cell 0 or the border cell under nearest)."""
    rng = np.random.default_rng(23)
    n, m, cin, cout = 60, 80, 3, 4
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    idx, rs, _ = O.c_radius(ip, op, 0.3)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    filt = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    nimp = rng.random(len(idx)).astype(np.float32)
    nimp[::5] = 0                                       # zero importance does not mask a non-finite feature
    f2 = feat.copy()
    f2[idx[3], 1], f2[idx[40], 0], f2[idx[90], 2] = np.nan, np.inf, -np.inf
    p2 = ip.copy()
    p2[idx[7], 0], p2[idx[60], 2] = np.nan, np.inf
    for pos, ft in ((ip, f2), (p2, feat)):
        args = (filt, op, [0.6], [0, 0, 0], pos, ft, None, idx, nimp, rs, mapping, interp, align, normalize)
        got, want = run_op(*args).cpu().numpy(), ref_op(*args)
        if pos is ip or interp == "linear":
            assert np.isnan(want).any()
        assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(np.isinf(got), np.isinf(want))
        assert np.array_equal(np.sign(got[np.isinf(got)]), np.sign(want[np.isinf(want)]))
        ok = np.isfinite(want)
        assert np.abs(got[ok] - want[ok]).max() < 1e-4 * np.abs(want[ok]).max()


# ------------------------------------------------------------------------------------------------------- refusals
def test_op_refusals():
    rng = np.random.default_rng(24)
    n, m, cin = 20, 15, 3
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    idx, rs = random_lists(rng, m, n, 3)

    def call(filt=np.zeros((2, 2, 2, cin, 4), np.float32), op=op, ip=ip, feat=feat, iimp=None, nimp=None, ext=(0.6,),
             mapping="identity", interp="linear", idx_dtype=torch.int64, rs=rs):
        return run_op(filt, op, list(ext), [0, 0, 0], ip, feat, iimp, idx, nimp, rs, mapping, interp, False, True,
                      index_dtype=idx_dtype)
    call()
    # short tensors the kernel would read by index
    with pytest.raises(RuntimeError, match="inp_importance must be empty or have 20 elements"):
        call(iimp=np.ones(n - 1, np.float32))
    with pytest.raises(RuntimeError, match="neighbors_importance must be empty or have %d elements" % len(idx)):
        call(nimp=np.ones(len(idx) - 1, np.float32))
    with pytest.raises(RuntimeError, match=r"inp_features must be \[num_inp, Cin\]"):
        call(feat=feat[:-1])
    with pytest.raises(RuntimeError, match=r"inp_features must be \[num_inp, Cin\]"):
        call(feat=feat[:, :2])
    with pytest.raises(RuntimeError, match=r"out_positions must have shape \[N, 3\]"):
        call(op=np.ascontiguousarray(op[:, :2]))
    with pytest.raises(RuntimeError, match=r"inp_positions must have shape \[N, 3\]"):
        call(ip=np.ascontiguousarray(ip[:, :2]))
    with pytest.raises(RuntimeError, match="extents must have 1 or num_out elements"):
        call(ext=(0.6,) * (m + 1))
    # shapes, options and index widths
    with pytest.raises(RuntimeError, match="out_channels <= 1024"):
        call(filt=np.zeros((1, 1, 1, cin, 1025), np.float32))
    with pytest.raises(RuntimeError, match="12288"):
        call(filt=np.zeros((1, 1, 1, 12289, 1), np.float32), feat=np.zeros((n, 12289), np.float32))
    with pytest.raises(RuntimeError, match="coordinate_mapping"):
        call(mapping="ball_to_cube_volume_preserving")
    with pytest.raises(RuntimeError, match="interpolation"):
        call(interp="cubic")
    with pytest.raises(RuntimeError, match="filters"):
        call(filt=np.zeros((2, 2, cin, 4), np.float32))
    with pytest.raises(RuntimeError, match="int32 or int64"):
        call(idx_dtype=torch.int16)
    with pytest.raises(RuntimeError, match="row_splits"):
        call(rs=rs[:-1])


# ------------------------------------------------------------------------------------------------------ the layer
@pytest.mark.parametrize("mapping,interp,align,normalize", GRID)
def test_layer_vs_oracle_search_and_op(mapping, interp, align, normalize):
    """One extent: the layer searches the inputs within extent / 2 of each output and runs the op; CPU in, CPU out."""
    rng = np.random.default_rng(25)
    n, m, cin, cout, ext = 600, 200, 6, 10, 0.5
    ip, op = rng.random((n, 3)).astype(np.float32), rng.random((m, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    with torch.no_grad():
        layer = LY.ContinuousConv(cin, cout, [3, 3, 3], align_corners=align, coordinate_mapping=mapping,
                                  interpolation=interp, normalize=normalize, use_bias=True).eval()
        layer.bias.normal_()
        out = layer(torch.from_numpy(feat), torch.from_numpy(ip), torch.from_numpy(op), ext)
    assert not out.is_cuda
    idx, rs, _ = O.c_radius(ip, op, ext / 2)
    want = ref_op(layer.kernel.detach().numpy(), op, [ext], [0, 0, 0], ip, feat, None, idx, None, rs, mapping, interp,
                  align, normalize) + layer.bias.detach().numpy()
    assert rel_err(out, want) < 1e-4
