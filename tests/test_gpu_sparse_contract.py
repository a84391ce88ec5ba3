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
