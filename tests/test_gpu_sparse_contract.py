"""The table mode of the tensor-core GEMM (o3dml_sparse_conv_tc, layers.contract_cells) against float64: channel counts
that are and are not multiples of 32, 27- and 8-cell tables, the BN-ReLU prologue on and off, row counts off the
128-row tile, no rows, and tiles whose rows are all shadow."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def reference(feat, table, w, pre=None, shift=None, residual=None):
    x = feat.double()
    if pre is not None:
        x = torch.relu(x * pre[0].double() + pre[1].double())
    xp = torch.cat([x, x.new_zeros(1, x.shape[1])])
    t = table.long().clamp(max=x.shape[0])
    t[t < 0] = x.shape[0]
    out = sum(xp[t[:, c]] @ w[c].double() for c in range(w.shape[0]))
    if shift is not None:
        out = out + shift.double()
    if residual is not None:
        out = out + residual.double()
    return out


def case(m, n, cin, cout, cells, shadow_frac, seed):
    g = torch.Generator().manual_seed(seed)
    table = torch.randint(0, n, (m, cells), generator=g, dtype=torch.int32)
    table[torch.rand(m, cells, generator=g) < shadow_frac] = n
    feat = torch.randn(n, cin, generator=g)
    w = torch.randn(cells, cin, cout, generator=g) / (cells * cin) ** 0.5
    pre = (0.5 + torch.rand(cin, generator=g), torch.rand(cin, generator=g) + 0.2)   # relu(shift) > 0: the trap
    return table, feat, w, pre


@pytest.mark.parametrize("cin", [3, 16, 32, 48, 224])
@pytest.mark.parametrize("cells", [27, 8])
@pytest.mark.parametrize("with_pre", [False, True])
def test_table_mode_vs_float64(cin, cells, with_pre):
    from open3d_ml_b200 import layers as LY
    m, n, cout = 1000 + 37, 900, 48
    table, feat, w, pre = case(m, n, cin, cout, cells, 0.6, seed=cin * 31 + cells)
    shift = torch.randn(cout)
    fd = LY.aligned_rows(feat.cuda())
    out = torch.full((m, cout), float("nan")).cuda()
    p = (pre[0].cuda(), pre[1].cuda()) if with_pre else None
    LY.contract_cells(fd, table.cuda(), LY.pack_cells(w), out, shift.cuda(), pre=p)
    ref = reference(feat, table, w, pre if with_pre else None, shift)
    err = float((out.cpu().double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err


def test_residual_strided_rows_and_leading_dimension():
    """Input and output as column slices of wider buffers, a residual, and a table whose row stride exceeds its cells."""
    from open3d_ml_b200 import layers as LY
    m, n, cin, cout = 300, 260, 32, 64
    table, feat, w, pre = case(m, n, cin, cout, 27, 0.3, seed=5)
    wide_in = torch.randn(n, 2 * cin).cuda()
    wide_in[:, cin:] = feat.cuda()
    wide_out = torch.zeros(m, 3 * cout).cuda()
    res = torch.randn(m, cout)
    tab = torch.full((m, 32), -1, dtype=torch.int32)
    tab[:, :27] = table
    LY.contract_cells(wide_in[:, cin:], tab.cuda()[:, :27], LY.pack_cells(w), wide_out[:, cout:2 * cout],
                      pre=(pre[0].cuda(), pre[1].cuda()), residual=res.cuda())
    ref = reference(feat, table, w, pre, None, res)
    err = float((wide_out[:, cout:2 * cout].cpu().double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err
    assert float(wide_out[:, :cout].abs().max()) == 0 and float(wide_out[:, 2 * cout:].abs().max()) == 0


def test_no_rows_and_all_shadow_rows():
    from open3d_ml_b200 import layers as LY
    n, cin, cout = 50, 48, 32
    feat = torch.randn(n, cin).cuda()
    w = LY.pack_cells(torch.randn(27, cin, cout))
    pre = (torch.ones(cin).cuda(), torch.full((cin,), 3.0).cuda())
    empty = torch.empty(0, cout).cuda()
    LY.contract_cells(feat, torch.empty(0, 27, dtype=torch.int32).cuda(), w, empty, pre=pre)
    # 300 rows (three tiles) whose every cell is shadow (n, or negative): the output is the shift alone
    table = torch.full((300, 27), n, dtype=torch.int32)
    table[::2] = -1
    shift = torch.randn(cout).cuda()
    out = torch.full((300, cout), float("nan")).cuda()
    LY.contract_cells(feat, table.cuda(), w, out, shift, pre=pre)
    assert torch.equal(out, shift.expand(300, cout))
    # one live row in the last tile only
    table[-1, 13] = 7
    LY.contract_cells(feat, table.cuda(), w, out, shift, pre=pre)
    assert torch.equal(out[:-1], shift.expand(299, cout))
    ref = torch.relu(feat[7].double() + 3.0) @ w.host.double().cuda()[13 * 64:13 * 64 + cin] + shift.double()
    assert float((out[-1].double() - ref).abs().max() / ref.abs().max()) < 1e-5


def test_refusals():
    from open3d_ml_b200 import layers as LY
    feat = torch.randn(10, 32).cuda()
    w = LY.pack_cells(torch.randn(27, 32, 16))
    out = torch.empty(4, 16).cuda()
    with pytest.raises(RuntimeError, match="weight image"):          # 8 cells against a 27-cell weight
        LY.contract_cells(feat, torch.zeros(4, 8, dtype=torch.int32).cuda(), w, out)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        LY.contract_cells(torch.randn(10, 35).cuda()[:, :32], torch.zeros(4, 27, dtype=torch.int32).cuda(), w, out)
    with pytest.raises(RuntimeError, match="kernel cells"):
        big = LY.pack_cells(torch.randn(513, 4, 16))
        LY.contract_cells(torch.randn(10, 4).cuda(), torch.zeros(4, 513, dtype=torch.int32).cuda(), big, out)


def expected_width(m, cout):
    """The column tile gemm_tc_launch picks for a table-mode product: 32 or 64 when the padded Cout is that, else
    128 unless the grid of 128-column tiles would fill at most half of the SMs."""
    from open3d_ml_b200 import _lib as L
    npad = L.pack_linear(torch.zeros(1, cout)).n_pad
    if npad <= 64:
        return npad
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 64 if 2 * ((m + 127) // 128) * (npad // 128) <= sms else 128


COLUMN_CASES = [(1, 300), (20, 3000), (33, 300), (65, 300), (65, 20000), (96, 9000), (129, 700), (129, 9000),
                (224, 8500), (768, 300), (768, 4000), (1536, 1100), (1536, 3000)]


def test_column_cases_reach_every_tile_width():
    assert {expected_width(m, cout) for cout, m in COLUMN_CASES} == {32, 64, 128}


@pytest.mark.parametrize("cout,m", COLUMN_CASES)
def test_column_tiles_vs_float64_and_deterministic(cout, m):
    from open3d_ml_b200 import layers as LY
    table, feat, w, pre = case(m, 700, 40, cout, 8, 0.5, seed=cout + m)
    fd, td, wp = LY.aligned_rows(feat.cuda()), table.cuda(), LY.pack_cells(w)
    p = (pre[0].cuda(), pre[1].cuda())
    out = torch.full((m, cout), float("nan")).cuda()
    LY.contract_cells(fd, td, wp, out, pre=p)
    ref = reference(feat.cuda(), td, w.cuda(), p)
    err = float((out.double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, (expected_width(m, cout), err)
    again = torch.empty_like(out)
    LY.contract_cells(fd, td, wp, again, pre=p)
    assert torch.equal(out, again)


def structured_table(tiles, n, cells, live, seed):
    """Tile t of 128 rows reads the cells live(t) (about half of its rows in each), nothing else."""
    g = torch.Generator().manual_seed(seed)
    table = torch.full((tiles * 128, cells), n, dtype=torch.int32)
    for t in range(tiles):
        for c in live(t):
            rows = torch.nonzero(torch.rand(128, generator=g) < 0.5).view(-1) + t * 128
            table[rows, c] = torch.randint(0, n, (len(rows),), generator=g, dtype=torch.int32)
    return table


@pytest.mark.parametrize("cin", [32, 64, 224])
@pytest.mark.parametrize("cout,tiles", [(48, 12), (200, 70)])
def test_structured_cell_skips(cin, cout, tiles):
    """Per 128-row tile: no cell, only the first, only the last, every other one, or the first k cells with k slices
    around the stage ring (4 stages at 128 columns, 6 below) and the 4-slice accumulator fold."""
    from open3d_ml_b200 import layers as LY
    cells, n = 27, 500
    spc = (cin + 31) // 32
    counts = sorted({max(1, s // spc) for s in (3, 4, 5, 6, 7, 8, 9)} | {k for k in (1, 2, 3)})
    patterns = [[], [0], [cells - 1], list(range(0, cells, 2))] + [list(range(k)) for k in counts]
    table = structured_table(tiles, n, cells, lambda t: patterns[t % len(patterns)], seed=cin + cout)
    g = torch.Generator().manual_seed(cin)
    feat = torch.randn(n, cin, generator=g)
    w = torch.randn(cells, cin, cout, generator=g) / (cells * cin) ** 0.5
    pre = (0.5 + torch.rand(cin, generator=g), torch.rand(cin, generator=g) + 0.2)
    shift = torch.randn(cout, generator=g)
    for p in (None, pre):
        pd = (p[0].cuda(), p[1].cuda()) if p is not None else None
        out = torch.full((len(table), cout), float("nan")).cuda()
        LY.contract_cells(LY.aligned_rows(feat.cuda()), table.cuda(), LY.pack_cells(w), out, shift.cuda(), pre=pd)
        ref = reference(feat.cuda(), table.cuda(), w.cuda(), pd, shift.cuda())
        assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-5
        assert torch.equal(out[:128], shift.cuda().expand(128, cout))           # tile 0 reads no cell


@pytest.mark.parametrize("cin", [4, 36, 100])
@pytest.mark.parametrize("with_pre", [False, True])
def test_zero_fill_past_cin(cin, with_pre):
    """NaN in the padding columns [Cin, ld) of every feature row and in the rows the table never names."""
    from open3d_ml_b200 import layers as LY
    m, n, cout = 400, 300, 24
    table, feat, w, pre = case(m, n - 40, cin, cout, 27, 0.4, seed=cin)
    table[table == n - 40] = n                        # shadow id: the row count of the NaN-padded buffer
    ld = (cin + 3) // 4 * 4 + 8
    buf = torch.full((n, ld), float("nan"))
    buf[:n - 40, :cin] = feat
    p = (pre[0].cuda(), pre[1].cuda()) if with_pre else None
    out = torch.empty(m, cout).cuda()
    LY.contract_cells(buf.cuda()[:, :cin], table.cuda(), LY.pack_cells(w), out, pre=p)
    ref = reference(feat.cuda(), table.cuda().clamp(max=n - 40), w.cuda(), p)
    assert not bool(out.isnan().any())
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-5


@pytest.mark.parametrize("act,slope", [("relu", 0.0), ("leaky", 0.1)])
@pytest.mark.parametrize("cout", [20, 37])
def test_scalar_store_epilogue(act, slope, cout):
    """out_ld and the residual stride not multiples of 4 and an output slice at an odd column (the scalar stores),
    with scale, shift, residual and relu / leaky; leaky through o3dml_sparse_conv_tc, whose slope is an argument."""
    from open3d_ml_b200 import _lib as L, layers as LY
    m, n, cin = 333, 200, 40
    table, feat, w, _ = case(m, n, cin, cout, 8, 0.3, seed=cout)
    g = torch.Generator().manual_seed(cout)
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    wide_res = torch.randn(m, cout + 3, generator=g).cuda()
    res = wide_res[:, 3:]
    wide_out = torch.zeros(m, cout + 6).cuda()
    out = wide_out[:, 1:1 + cout]
    fd, td, wp = LY.aligned_rows(feat.cuda()), table.cuda(), LY.pack_cells(w)
    sd, hd = scale.cuda(), shift.cuda()
    L.check(L.lib().o3dml_sparse_conv_tc(
        m, L.ptr(fd), n, cin, fd.stride(0), L.ptr(td), 8, td.stride(0), None, None, L.ptr(wp.img), wp.k_pad, wp.n_pad,
        L.ptr(sd), L.ptr(hd), L.ptr(res), res.stride(0), L.act_code(act), slope, L.ptr(out),
        out.stride(0), cout, L.stream()))
    x = reference(feat.cuda(), td, w.cuda()) * sd.double() + hd.double() + res.double()
    ref = torch.where(x >= 0, x, x * slope)
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-5
    assert float(wide_out[:, :1].abs().max()) == 0 and float(wide_out[:, 1 + cout:].abs().max()) == 0
