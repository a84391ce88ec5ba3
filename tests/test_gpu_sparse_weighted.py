"""The weighted sparse convolution against float64: the raw ops.sparse_conv with importances and
ops.sparse_conv_transpose on ragged lists (repeated cells, rows whose every cell repeats, empty rows), the weighted
contraction's exactness (unit, power-of-two and zero weights, the weight after the BN-ReLU prologue), the adjoint
identity of the pair, the layers' inp_importance / out_importance, the refusals and the host reads."""
import warnings

import numpy as np
import pytest
import torch

from sparse_tables_support import brute_table, contract64
from test_gpu_sparse_tables import lattice, ragged_case

pytestmark = pytest.mark.gpu


def importance(kind, n, rng):
    """Dyadic values (multiples of 1/8), so that products and sums of a few of them are exact in float32 and a
    normalising divisor is the same in float32 and float64."""
    if kind == "empty":
        return None
    if kind == "zero":
        return np.zeros(n)
    if kind == "pos":
        return rng.integers(1, 17, n) / 8.0
    if kind == "neg":
        return -rng.integers(1, 17, n) / 8.0
    return rng.integers(-16, 17, n) / 8.0       # "signed", zeros included


def tensor(a):
    return torch.empty(0) if a is None else torch.from_numpy(np.asarray(a, np.float32)).cuda()


def ref_sparse_conv(feat, w, nidx, kidx, rs, iimp, nimp, normalize):
    """float64 out[o] = (1 / n_o) sum_e nimp_e iimp_i W[k_e]^T f[i]."""
    e = len(nidx)
    wt = (np.ones(e) if nimp is None else nimp) * (1.0 if iimp is None else iimp[nidx])
    rows = np.repeat(np.arange(len(rs) - 1), np.diff(rs))
    contrib = np.zeros((e, w.shape[2]))
    for c in range(w.shape[0]):
        sel = kidx == c
        contrib[sel] = (wt[sel, None] * feat[nidx[sel]].astype(np.float64)) @ w[c]
    out = np.zeros((len(rs) - 1, w.shape[2]))
    np.add.at(out, rows, contrib)
    if normalize:
        n_o = np.zeros(len(rs) - 1)
        np.add.at(n_o, rows, wt)
        out /= np.where(n_o != 0, n_o, 1.0)[:, None]
    return out


def ref_sparse_conv_transpose(feat, w, nidx, kidx, rs, oimp, nimp, s):
    """float64 out[j] = oimp_j sum_e nimp_e s_i W[k_e]^T f[i] (s None: ones)."""
    nimp2 = (np.ones(len(nidx)) if nimp is None else nimp) * (1.0 if s is None else s[nidx])
    out = ref_sparse_conv(feat, w, nidx, kidx, rs, None, nimp2, False)
    return out if oimp is None else out * oimp[:, None]


def rel_check(got, ref, tol=1e-5):
    got = got.cpu().double().numpy()
    scale = np.abs(ref).max()
    if scale == 0:
        assert np.abs(got).max() == 0
    else:
        assert float(np.abs(got - ref).max() / scale) < tol


IMPORTANCE_PAIRS = [("empty", "empty"), ("pos", "empty"), ("empty", "pos"), ("pos", "pos"), ("zero", "pos"),
                    ("pos", "zero"), ("neg", "signed"), ("signed", "neg"), ("empty", "signed")]


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("ikind,nkind", IMPORTANCE_PAIRS)
def test_raw_sparse_conv_importance(dtype, normalize, ikind, nkind):
    import open3d_ml_b200 as M
    nidx, kidx, rs = ragged_case(3)
    rng = np.random.default_rng(4)
    cin, cout, n = 24, 40, 300
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    k = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    w = k.reshape(27, cin, cout).astype(np.float64)
    iimp, nimp = importance(ikind, n, rng), importance(nkind, len(nidx), rng)
    if nimp is not None and nkind == "signed":          # row 5 (distinct cells) sums to zero
        a, b = rs[5], rs[6]
        nimp[a:b] = [(1.0 if j % 2 == 0 else -1.0) for j in range(b - a)]
        if (b - a) % 2:
            nimp[b - 1] = 0.0
    args = (torch.from_numpy(k), torch.from_numpy(feat).cuda(), tensor(iimp), torch.from_numpy(nidx).to(dtype).cuda(),
            torch.from_numpy(kidx).cuda(), tensor(nimp), torch.from_numpy(rs).cuda(), normalize)
    got = M.ops.sparse_conv(*args)
    ref = ref_sparse_conv(feat, w, nidx, kidx, rs, iimp, nimp, normalize)
    rel_check(got, ref)
    assert torch.equal(got, M.ops.sparse_conv(*args))
    assert float(got[0::4].abs().max()) == 0


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("norm", [None, "sum", "splits"])
@pytest.mark.parametrize("okind,nkind", [("empty", "empty"), ("pos", "pos"), ("neg", "signed"), ("zero", "pos"),
                                         ("signed", "empty")])
def test_raw_sparse_conv_transpose(dtype, norm, okind, nkind):
    import open3d_ml_b200 as M
    nidx, kidx, rs = ragged_case(5)
    rng = np.random.default_rng(6)
    cin, cout, n = 36, 20, 300
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    k = rng.standard_normal((27, cin, cout)).astype(np.float32)
    oimp, nimp = importance(okind, len(rs) - 1, rng), importance(nkind, len(nidx), rng)
    isum, irs, s = None, None, None
    if norm == "sum":
        isum = rng.integers(-8, 9, n) / 4.0                                   # zeros included: divisor 1
        s = np.where(isum != 0, 1.0 / np.where(isum != 0, isum, 1.0), 1.0)
    elif norm == "splits":
        irs = np.concatenate([[0], np.cumsum(rng.integers(0, 4, n))]).astype(np.int64)
        ln = np.diff(irs).astype(np.float64)
        s = np.where(ln != 0, 1.0 / np.where(ln != 0, ln, 1.0), 1.0)
    got = M.ops.sparse_conv_transpose(
        torch.from_numpy(k), tensor(oimp), torch.from_numpy(feat).cuda(), torch.empty(0), tensor(isum),
        torch.empty(0, dtype=torch.int64) if irs is None else torch.from_numpy(irs).cuda(),
        torch.from_numpy(nidx).to(dtype).cuda(), torch.from_numpy(kidx).cuda(), tensor(nimp),
        torch.from_numpy(rs).cuda(), normalize=norm is not None)
    ref = ref_sparse_conv_transpose(feat, k.astype(np.float64), nidx, kidx, rs, oimp, nimp, s)
    rel_check(got, ref)


def table_case(m, n, cin, cells, shadow, seed):
    g = torch.Generator().manual_seed(seed)
    table = torch.randint(0, n, (m, cells), generator=g, dtype=torch.int32)
    table[torch.rand(m, cells, generator=g) < shadow] = n
    feat = torch.randn(n, cin, generator=g)
    w = torch.randn(cells, cin, 48, generator=g) / (cells * cin) ** 0.5
    pre = (0.5 + torch.rand(cin, generator=g), torch.rand(cin, generator=g) - 0.4)
    return table, feat, w, pre


@pytest.mark.parametrize("cin", [3, 32, 48])
@pytest.mark.parametrize("cells", [27, 8])
@pytest.mark.parametrize("with_pre", [False, True])
def test_weight_path_exactness(cin, cells, with_pre):
    """Unit weights reproduce the unweighted entry bit for bit, 2^-3 scales it exactly, a zero weight on a live entry
    equals a shadow entry, and the weight multiplies after the prologue (float64 with negative weights)."""
    from open3d_ml_b200 import layers as LY
    m, n = 700 + 37, 500
    table, feat, w, pre = table_case(m, n, cin, cells, 0.3, seed=cin * 7 + cells)
    fd, td, wp = LY.aligned_rows(feat.cuda()), table.cuda(), LY.pack_cells(w)
    p = (pre[0].cuda(), pre[1].cuda()) if with_pre else None

    def run(tab, weight=None):
        out = torch.full((m, 48), float("nan")).cuda()
        return LY.contract_cells(fd, tab, wp, out, pre=p, entry_weight=weight)
    plain = run(td)
    ones = torch.ones(m, cells).cuda()
    assert torch.equal(run(td, ones), plain)
    assert torch.equal(run(td, ones * 0.125), plain * 0.125)
    g = torch.Generator().manual_seed(cin)
    drop = (torch.rand(m, cells, generator=g) < 0.3).cuda() & (td < n)
    zeroed = run(td, torch.where(drop, 0.0, 1.0))
    assert torch.equal(zeroed, run(torch.where(drop, n, td)))
    # signed weights, NaN on the shadow entries: the weight applies after the prologue and shadows stay zero
    wt = torch.randn(m, cells, generator=g).cuda()
    wt[td >= n] = float("nan")
    got = run(td, wt)
    x = feat.cuda().double()
    if with_pre:
        x = torch.relu(x * p[0].double() + p[1].double())
    xp = torch.cat([x, x.new_zeros(1, cin)])
    tl = td.long()
    wd = torch.where(td < n, wt, 0.0).double()
    ref = sum((wd[:, c:c + 1] * xp[tl[:, c]]) @ w[c].cuda().double() for c in range(cells))
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < 1e-5


@pytest.mark.parametrize("normalize", [False, True])
def test_adjoint_identity(normalize):
    """sum_i <z_i, x_i> = sum_j <y_j, T(x)_j>: T the transposed op on lists (rows = its outputs), z the forward op on
    the inverted lists (kernel index and importance carried by invert_neighbors_list) with the filters transposed per
    cell and inp_importance = out_importance; under normalize T takes inp_neighbors_importance_sum[i] = sum over the
    inverted row i of nimp_e * oimp_j, the divisor the forward computes."""
    import open3d_ml_b200 as M
    nidx, kidx, rs = ragged_case(8, n=250, rows=300)
    rng = np.random.default_rng(9)
    cin, cout, n_in, n_out = 20, 28, 250, 300
    k = torch.from_numpy(rng.standard_normal((27, cin, cout)).astype(np.float32))
    x = torch.from_numpy(rng.standard_normal((n_in, cin)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.standard_normal((n_out, cout)).astype(np.float32)).cuda()
    oimp, nimp = tensor(rng.integers(1, 17, n_out) / 8.0), tensor(rng.integers(-16, 17, len(nidx)) / 8.0)
    idx, kc, splits = torch.from_numpy(nidx).cuda(), torch.from_numpy(kidx).cuda(), torch.from_numpy(rs).cuda()
    inv_k = M.ops.invert_neighbors_list(n_in, idx, splits, kc)
    inv_w = M.ops.invert_neighbors_list(n_in, idx, splits, nimp)
    rows = torch.repeat_interleave(torch.arange(n_out).cuda(), splits[1:] - splits[:-1])
    isum = torch.zeros(n_in, dtype=torch.float64).cuda().index_add_(0, idx.long(), nimp.double() * oimp.double()[rows])
    t = M.ops.sparse_conv_transpose(k, oimp, x, torch.empty(0), isum.float(), torch.empty(0, dtype=torch.int64), idx, kc,
                                    nimp, splits, normalize=normalize)
    z = M.ops.sparse_conv(k.transpose(-1, -2), y, oimp, inv_k.neighbors_index, inv_k.neighbors_attributes,
                          inv_w.neighbors_attributes, inv_k.neighbors_row_splits, normalize=normalize)
    lhs = float((z.double() * x.double()).sum())
    rhs = float((y.double() * t.double()).sum())
    scale = float((z.double() * x.double()).abs().sum())
    assert abs(lhs - rhs) < 1e-5 * scale, (lhs, rhs, scale)


@pytest.mark.parametrize("layer", ["SparseConv", "SparseConvTranspose"])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("bias", [False, True])
def test_layers_with_importance(layer, normalize, bias):
    from open3d_ml_b200 import layers as LY
    rng = np.random.default_rng(11)
    v, inp, out = 1.0, lattice(2000, 16, 10) + 0.9, lattice(1200, 16, 11) + 0.1
    inp, out = inp.astype(np.float32), out.astype(np.float32)
    cin, cout, ks = 12, 20, [3, 3, 3]
    transpose = layer == "SparseConvTranspose"
    feat = rng.standard_normal((len(inp), cin)).astype(np.float32)
    imp = (rng.integers(-16, 17, len(out) if transpose else len(inp)) / 8.0).astype(np.float32)
    torch.manual_seed(1)
    with torch.no_grad():
        conv = getattr(LY, layer)(cin, cout, ks, normalize=normalize, use_bias=bias, offset=torch.zeros(3)).eval()
        if bias:
            conv.bias.normal_()
        args = (torch.from_numpy(feat).cuda(), torch.from_numpy(inp).cuda(), torch.from_numpy(out).cuda(), v)
        key = "out_importance" if transpose else "inp_importance"
        got = conv(*args, **{key: torch.from_numpy(imp).cuda()})
        plain = conv(*args)
        ones = conv(*args, **{key: torch.ones(len(imp)).cuda()})
    assert torch.equal(plain, ones)
    table, cnt = brute_table(inp, out, v, [0, 0, 0], ks, transpose)
    kernel = conv.kernel.detach().numpy()
    if transpose:
        ref = contract64(feat, table, kernel) * imp[:, None]
    else:
        ref = contract64(feat * imp[:, None].astype(np.float64), table, kernel)
    if normalize:
        ref = ref / np.maximum(cnt, 1)[:, None]
    if bias:
        ref = ref + conv.bias.detach().numpy()
    rel_check(got, ref)


def test_refusals_before_any_launch():
    import open3d_ml_b200 as M
    from open3d_ml_b200 import _lib as L, layers as LY
    nidx, kidx, rs = ragged_case(12, n=50, rows=40)
    k = torch.randn(27, 8, 16)
    feat = torch.randn(50, 8).cuda()
    idx, kc, splits = torch.from_numpy(nidx).cuda(), torch.from_numpy(kidx).cuda(), torch.from_numpy(rs).cuda()
    e = len(nidx)

    def refused(match, call):
        torch.cuda.synchronize()
        n0 = L.lib().o3dml_launch_count()
        with pytest.raises(RuntimeError, match=match):
            call()
        assert L.lib().o3dml_launch_count() == n0

    for bad in (27, -1):
        kb = kc.clone()
        kb[e // 2] = bad
        refused("neighbors_kernel_index", lambda: M.ops.sparse_conv(k, feat, torch.empty(0), idx, kb, torch.empty(0),
                                                                     splits))
        refused("neighbors_kernel_index", lambda: M.ops.sparse_conv_transpose(
            k, torch.empty(0), feat, torch.empty(0), torch.empty(0), torch.empty(0), idx, kb, torch.empty(0), splits))
    refused("inp_importance", lambda: M.ops.sparse_conv(k, feat, torch.ones(49).cuda(), idx, kc, torch.empty(0), splits))
    refused("neighbors_importance", lambda: M.ops.sparse_conv(k, feat, torch.empty(0), idx, kc,
                                                              torch.ones(e + 1).cuda(), splits))
    refused("out_importance", lambda: M.ops.sparse_conv_transpose(
        k, torch.ones(len(rs)).cuda(), feat, torch.empty(0), torch.empty(0), torch.empty(0), idx, kc, torch.empty(0),
        splits))
    refused("inp_neighbors_importance_sum", lambda: M.ops.sparse_conv_transpose(
        k, torch.empty(0), feat, torch.empty(0), torch.ones(49).cuda(), torch.empty(0), idx, kc, torch.empty(0), splits,
        normalize=True))
    refused("normalize needs", lambda: M.ops.sparse_conv_transpose(
        k, torch.empty(0), feat, torch.empty(0), torch.empty(0), torch.empty(0), idx, kc, torch.empty(0), splits,
        normalize=True))
    pos = torch.from_numpy(lattice(60, 6, 3).astype(np.float32)).cuda()
    with torch.no_grad():
        conv, up = LY.SparseConv(8, 16, [3, 3, 3]), LY.SparseConvTranspose(8, 16, [3, 3, 3])
        f = torch.randn(len(pos), 8).cuda()
        refused("inp_importance", lambda: conv(f, pos, pos, 1.0, inp_importance=torch.ones(len(pos) + 1).cuda()))
        refused("out_importance", lambda: up(f, pos, pos, 1.0, out_importance=torch.ones(len(pos) - 1).cuda()))
        refused("user neighbours", lambda: up(f, pos, pos, 1.0, user_neighbors_index=torch.zeros(3).cuda()))


def syncs(call):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            call()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return [str(x.message) for x in w if "synchroniz" in str(x.message)]


def test_host_reads(monkeypatch):
    """One host read per raw-op call (the filters are packed outside the count: that is a host-to-device copy), and
    importance adds none to the layers."""
    import open3d_ml_b200 as M
    from open3d_ml_b200 import layers as LY
    nidx, kidx, rs = ragged_case(13)
    k = torch.randn(27, 16, 24)
    feat = torch.randn(300, 16).cuda()
    idx, kc, splits = torch.from_numpy(nidx).cuda(), torch.from_numpy(kidx).cuda(), torch.from_numpy(rs).cuda()
    iimp, nimp, oimp = torch.rand(300).cuda(), torch.rand(len(nidx)).cuda(), torch.rand(len(rs) - 1).cuda()
    packed, pack = {}, LY.pack_cells

    def pack_cells(w):
        key = tuple(w.shape)
        if key not in packed:
            packed[key] = pack(w)
        return packed[key]
    monkeypatch.setattr(LY, "pack_cells", pack_cells)
    calls = [lambda: M.ops.sparse_conv(k, feat, iimp, idx, kc, nimp, splits, True),
             lambda: M.ops.sparse_conv_transpose(k, oimp, feat, torch.empty(0), torch.empty(0), splits, idx, kc, nimp,
                                                 splits, False)]
    for call in calls:
        call()                                   # packs the filters
        got = syncs(call)
        assert len(got) == 1, got
    monkeypatch.undo()
    pos = torch.from_numpy(lattice(800, 12, 4).astype(np.float32)).cuda()
    f = torch.randn(len(pos), 16).cuda()
    with torch.no_grad():
        for layer, key in ((LY.SparseConv, "inp_importance"), (LY.SparseConvTranspose, "out_importance")):
            conv = layer(16, 24, [3, 3, 3], normalize=True)
            imp = torch.rand(len(pos)).cuda()
            conv(f, pos, pos, 1.0)                       # packs the kernel
            assert len(syncs(lambda: conv(f, pos, pos, 1.0, **{key: imp}))) == len(syncs(lambda: conv(f, pos, pos, 1.0)))
