"""The neighbour tables of the sparse convolutions (o3dml_sparse_conv_neighbors) against a brute-force float32 table
over every (output, input) pair (sparse_tables_support.brute_table, pinned to the oracle in tests/test_oracle_ops.py):
positions off the voxel grid, at voxel corners out to 2e4 cells, beyond the 2^20-cell key fields, every kernel shape
and offset, empty sides, and points on cell faces where a fused multiply-add would change the cell.  Then the layers
and the raw ops.sparse_conv (rows that name one kernel cell several times) against float64."""
import numpy as np
import pytest
import torch

from sparse_tables_support import brute_table, contract64, face_points

pytestmark = pytest.mark.gpu


def check(inp, out, v, offset, ks, transpose=False):
    from open3d_ml_b200 import layers as LY
    inp, out = np.asarray(inp, np.float32).reshape(-1, 3), np.asarray(out, np.float32).reshape(-1, 3)
    want, want_cnt = brute_table(inp, out, v, offset, ks, transpose)
    nbr, cnt = LY.sparse_conv_neighbors(torch.from_numpy(inp), torch.from_numpy(out), v, list(offset), ks, transpose,
                                        want_count=True)
    got = nbr.cpu().numpy()
    bad = int((got != want).sum())
    assert bad == 0, "%d of %d table entries differ (%d neighbours expected)" % (bad, want.size, int((want < len(inp)).sum()))
    assert np.array_equal(cnt.cpu().numpy(), want_cnt)
    return want


def lattice(n, extent, seed, base=0):
    """Voxel-unique integer cells: n draws in [0, extent)^3 shifted by base."""
    rng = np.random.default_rng(seed)
    return np.unique(rng.integers(0, extent, (n, 3)), axis=0) + np.asarray(base, np.int64)


@pytest.mark.parametrize("fi,fo", [(0.5, 0.5), (0.9, 0.1), (0.25, 0.75), (0.0, 0.0)])
@pytest.mark.parametrize("ks,off", [((3, 3, 3), 0.0), ((2, 2, 2), -0.5)])
def test_grid_alignment(fi, fo, ks, off):
    """Inputs at k + fi, outputs at k + fo (voxel 1): a cell box straddles two input voxels unless fi = fo."""
    inp = lattice(2500, 18, 1) + fi
    out = lattice(1500, 18, 2) + fo
    t = check(inp, out, 1.0, [off] * 3, ks)
    assert (t < len(inp)).sum() > 1000


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("v", [1.0, 0.3])
def test_uniform_clouds_lowest_id(v, transpose):
    """Several inputs per cell: the table keeps the lowest id."""
    rng = np.random.default_rng(3)
    inp = (rng.random((3000, 3)) * 8 * v).astype(np.float32)
    out = (rng.random((800, 3)) * 8 * v).astype(np.float32)
    t = check(inp, out, v, [0.0] * 3, [3, 3, 3], transpose)
    assert (t < len(inp)).mean() > 0.5
    check(inp, out, v, [-0.5] * 3, [2, 2, 2], transpose)


@pytest.mark.parametrize("v", [1.0, 0.5, 0.05, 0.02, 0.3])
@pytest.mark.parametrize("frac", [0.0, 0.5])
def test_voxel_sizes_corners_and_centres_far_out(v, frac):
    """Positions (k + frac) * v with k out to 2e4 cells, in clusters so that the tables are dense."""
    rng = np.random.default_rng(4)
    inp, out = [], []
    for i, base in enumerate(rng.integers(-20000, 20000, (4, 3))):
        inp.append(lattice(600, 10, 10 + i, base))
        out.append(lattice(300, 10, 20 + i, base))
    inp = ((np.concatenate(inp) + frac) * np.float32(v)).astype(np.float32)
    out = ((np.concatenate(out) + frac) * np.float32(v)).astype(np.float32)
    t = check(inp, out, v, [0.0] * 3, [3, 3, 3])
    assert (t < len(inp)).sum() > 1000
    check(inp, out, v, [-0.5] * 3, [2, 2, 2], transpose=True)


@pytest.mark.parametrize("v", [1.0, 0.5])
def test_negative_and_beyond_the_key_fields(v):
    """Cells below zero and past +-2^20, where the 21-bit fields of the voxel key alias: never a lost neighbour."""
    far = 1 << 20
    inp, out = [], []
    for i, base in enumerate([(-30, -5, -12), (far + 100, 3, -far - 50), (-far - 300, far + 7, 5), (far - 4, -far + 2, 0)]):
        inp.append(lattice(500, 9, 30 + i, base))
        out.append(lattice(300, 9, 40 + i, base))
    for fi, fo in ((0.5, 0.5), (0.75, 0.25)):
        ip = ((np.concatenate(inp) + fi) * v).astype(np.float32)
        op = ((np.concatenate(out) + fo) * v).astype(np.float32)
        t = check(ip, op, v, [0.0] * 3, [3, 3, 3])
        assert (t < len(ip)).sum() > 500


@pytest.mark.parametrize("ks", [(1, 1, 1), (2, 2, 2), (3, 3, 3), (4, 4, 4), (5, 5, 5), (9, 9, 9), (1, 3, 5), (2, 3, 4)])
def test_kernel_sizes(ks):
    rng = np.random.default_rng(5)
    inp = (lattice(2000, 14, 6) + rng.random((1, 3))).astype(np.float32)
    out = (rng.random((300, 3)) * 14).astype(np.float32)
    off = [0.0 if k % 2 else -0.5 for k in ks]
    check(inp, out, 1.0, off, ks)
    check(inp, out, 0.7, [0.25, -0.25, 0.0], ks, transpose=True)


@pytest.mark.parametrize("off", [0.0, -0.5, 0.25, -0.25])
@pytest.mark.parametrize("transpose", [False, True])
def test_offsets(off, transpose):
    rng = np.random.default_rng(7)
    inp = (lattice(2000, 14, 8) + 0.3).astype(np.float32)
    out = (rng.random((600, 3)) * 14).astype(np.float32)
    check(inp, out, 1.0, [off] * 3, [3, 3, 3], transpose)
    check(inp * 0.05, out * 0.05, 0.05, [off, 0.0, -off], [2, 3, 2], transpose)


def test_empty_sides_and_one_input():
    p = np.array([[0.5, 0.5, 0.5], [1.5, 0.5, 0.5], [9.0, 9.0, 9.0]], np.float32)
    check(p[:0], p, 1.0, [0.0] * 3, [3, 3, 3])
    check(p, p[:0], 1.0, [0.0] * 3, [3, 3, 3])
    t = check(p[:1], p, 1.0, [0.0] * 3, [3, 3, 3])
    assert t[0, 13] == 0 and t[1, 4] == 0 and (t[2] == 1).all()


@pytest.mark.parametrize("v,off,ks,transpose", [(0.05, -0.5, 2, True), (0.02, -0.25, 3, False), (0.3, -0.5, 4, True),
                                                (0.05, 0.25, 2, True), (0.3, -0.25, 3, False)])
def test_points_on_cell_faces(v, off, ks, transpose):
    """Inputs on the faces of the cells, where fusing the product into the offset add moves the point to the next
    cell: the table follows the unfused rounding of the oracle."""
    pairs = face_points(v, off, ks, transpose, 64, seed=ks)
    assert pairs, "no point where the fused and the unfused predicate disagree"
    inp, out = [], []
    for i, (a, b) in enumerate(pairs):
        y = np.float32(i * 40 * v)                      # one pair per row of the lattice, far from the others
        inp.append((a, y, 0.0))
        out.append((b, y, 0.0))
    check(inp, out, v, [off, 0.0, 0.0], (ks, 1, 1), transpose)


@pytest.mark.parametrize("layer", ["SparseConv", "SparseConvTranspose"])
@pytest.mark.parametrize("case", ["off_grid", "corner"])
def test_layers_off_the_grid(layer, case):
    """The drop-in layers with normalize and bias against the brute-force table contracted in float64."""
    from open3d_ml_b200 import layers as LY
    rng = np.random.default_rng(9)
    if case == "off_grid":
        v, inp, out = 1.0, lattice(2000, 16, 10) + 0.9, lattice(1200, 16, 11) + 0.1
    else:
        v = 0.05
        inp, out = (lattice(2000, 16, 12, 15000) * v), (lattice(1200, 16, 13, 15000) * v)
    inp, out = inp.astype(np.float32), out.astype(np.float32)
    cin, cout, ks = 12, 20, [3, 3, 3]
    feat = rng.standard_normal((len(inp), cin)).astype(np.float32)
    torch.manual_seed(0)
    with torch.no_grad():
        conv = getattr(LY, layer)(cin, cout, ks, normalize=True, offset=torch.zeros(3)).eval()
        conv.bias.normal_()
        got = conv(torch.from_numpy(feat).cuda(), torch.from_numpy(inp).cuda(), torch.from_numpy(out).cuda(), v)
    table, cnt = brute_table(inp, out, v, [0, 0, 0], ks, layer == "SparseConvTranspose")
    assert (cnt > 1).mean() > 0.5
    kernel, bias = conv.kernel.detach().numpy(), conv.bias.detach().numpy()
    ref = contract64(feat, table, kernel) / np.maximum(cnt, 1)[:, None] + bias
    assert float(np.abs(got.cpu().numpy() - ref).max() / np.abs(ref).max()) < 1e-5


def ragged_case(seed, n=300, rows=400, kc=27):
    """Ragged (index, kernel cell) lists: rows that repeat cells, rows whose every cell is repeated, empty rows."""
    rng = np.random.default_rng(seed)
    nidx, kidx, rs = [], [], [0]
    for r in range(rows):
        kind = r % 4
        if kind == 0:                                   # empty
            cells = []
        elif kind == 1:                                 # distinct cells
            cells = list(rng.choice(kc, rng.integers(1, kc), replace=False))
        elif kind == 2:                                 # some cells repeated
            cells = list(rng.integers(0, kc, rng.integers(5, 40)))
        else:                                           # every cell repeated, up to four times
            base = list(rng.choice(kc, rng.integers(1, 6), replace=False))
            cells = [c for c in base for _ in range(rng.integers(2, 5))]
            rng.shuffle(cells)
        nidx += list(rng.integers(0, n, len(cells)))
        kidx += cells
        rs.append(len(nidx))
    return np.array(nidx), np.array(kidx), np.array(rs, np.int64)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("normalize", [False, True])
def test_raw_sparse_conv_repeated_cells(dtype, normalize):
    """ops.sparse_conv sums every entry of a row, also when a row names one kernel cell more than once."""
    import open3d_ml_b200 as M
    nidx, kidx, rs = ragged_case(1)
    rng = np.random.default_rng(2)
    cin, cout = 24, 40
    feat = rng.standard_normal((300, cin)).astype(np.float32)
    k = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    w = k.reshape(27, cin, cout).astype(np.float64)
    ref = np.zeros((len(rs) - 1, cout))
    for r in range(len(rs) - 1):
        for j in range(rs[r], rs[r + 1]):
            ref[r] += feat[nidx[j]].astype(np.float64) @ w[kidx[j]]
        if normalize and rs[r + 1] > rs[r]:
            ref[r] /= rs[r + 1] - rs[r]
    args = (torch.from_numpy(k), torch.from_numpy(feat).cuda(), torch.empty(0), torch.from_numpy(nidx).to(dtype).cuda(),
            torch.from_numpy(kidx).cuda(), torch.empty(0), torch.from_numpy(rs).cuda(), normalize)
    got = M.ops.sparse_conv(*args)
    assert float((got.cpu().double() - torch.from_numpy(ref)).abs().max() / np.abs(ref).max()) < 1e-5
    assert torch.equal(got, M.ops.sparse_conv(*args))
    assert float(got[0::4].abs().max()) == 0
