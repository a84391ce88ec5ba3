"""The op oracle pinned against itself (C brute force vs numpy/KD-tree), against
scipy / sklearn KD-trees, and against hand-computable cases (parity is otherwise
UNPINNED by the reference: SURVEY.md 8c)."""
import numpy as np
import pytest

from oracle import ops as O
from open3d_ml_b200 import synth
from cconv_cases import far_neighbours

KITTI = dict(voxel_size=[0.16, 0.16, 4], range_min=[0, -39.68, -3], range_max=[69.12, 39.68, 1])


def test_voxelize_c_vs_numpy_and_invariants():
    pts = synth.lidar_frame(20000, 3)[:, :3]
    pts[:7, 0] = 69.12      # p == max is kept and yields index == extent (SURVEY A3)
    pts[7:11, 1] = 39.68
    pts[11:20, 2] = 5.0     # out of range
    a = O.c_voxelize(pts, None, KITTI["voxel_size"], KITTI["range_min"], KITTI["range_max"], 32, 40000)
    b = O.np_voxelize(pts, None, KITTI["voxel_size"], KITTI["range_min"], KITTI["range_max"], 32, 40000)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    c, rs, pi = a["voxel_coords"], a["voxel_point_row_splits"], a["voxel_point_indices"]
    assert c[:, 0].max() == 432 and c[:, 1].max() == 496
    lin = c[:, 0].astype(np.int64) + 1000 * (c[:, 1] + 1000 * c[:, 2].astype(np.int64))
    assert np.all(np.diff(lin) > 0)                      # voxels ascend, unique
    assert np.all(np.diff(rs) >= 1) and np.all(np.diff(rs) <= 32)
    for v in range(0, len(rs) - 1, 97):
        ids = pi[rs[v]:rs[v + 1]]
        assert np.all(np.diff(ids) > 0)                  # ids ascend inside a voxel
        ijk = ((pts[ids] - np.float32(KITTI["range_min"])) * (np.float32(1) / np.float32(KITTI["voxel_size"]))).astype(np.int64)
        assert np.all(ijk == c[v])
    assert not np.isin(np.arange(11, 20), pi).any()


def test_voxelize_caps_and_batch():
    rng = np.random.default_rng(0)
    pts = rng.uniform(0, 1, (10000, 3)).astype(np.float32)   # reference smoke test shape (test_models.py:204-236)
    a = O.c_voxelize(pts, [0, 4000, 4000, 10000], [0.16, 0.16, 4], [0, -39.68, -3], [69.12, 39.68, 1], 32, 20)
    b = O.np_voxelize(pts, [0, 4000, 4000, 10000], [0.16, 0.16, 4], [0, -39.68, -3], [69.12, 39.68, 1], 32, 20)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    assert list(a["voxel_batch_splits"]) == [0, 20, 20, 40]
    assert np.diff(a["voxel_point_row_splits"]).max() == 32
    # first 32 ids of the first voxel of batch 0 are the 32 smallest ids in that cell
    cell0 = a["voxel_coords"][0]
    ijk = (pts[:4000] * (np.float32(1) / np.float32([0.16, 0.16, 4]))).astype(np.int64)
    ijk[:, 1] = ((pts[:4000, 1] + np.float32(39.68)) * (np.float32(1) / np.float32(0.16))).astype(np.int64)
    ijk[:, 2] = ((pts[:4000, 2] + np.float32(3)) * np.float32(0.25)).astype(np.int64)
    members = np.nonzero(np.all(ijk == cell0, axis=1))[0]
    assert np.array_equal(a["voxel_point_indices"][:32], members[:32])


def test_voxelize_empty():
    a = O.c_voxelize(np.zeros((0, 3), np.float32), None, [1, 1, 1], [0, 0, 0], [4, 4, 4])
    assert a["voxel_coords"].shape == (0, 3) and list(a["voxel_point_row_splits"]) == [0]


def test_ragged_to_dense():
    v = np.arange(10, dtype=np.int64)
    out = O.np_ragged_to_dense(v, [0, 3, 3, 10], 4, -1)
    assert out.tolist() == [[0, 1, 2, -1], [-1, -1, -1, -1], [3, 4, 5, 6]]


@pytest.mark.parametrize("gen", ["uniform", "lidar"])
def test_knn_c_vs_numpy_vs_kdtree(gen):
    from scipy.spatial import cKDTree
    from sklearn.neighbors import KDTree
    P = synth.uniform_cloud(6000, 1) if gen == "uniform" else synth.semantickitti_cloud(6000, 1)
    i1, d1 = O.c_knn(P, P, 16)
    i2, d2 = O.np_knn(P, P, 16)
    assert np.array_equal(i1, i2) and np.array_equal(d1, d2)
    assert np.array_equal(i1[:, 0], np.arange(len(P)))            # self first
    assert np.all(np.diff(d1, axis=1) >= 0)
    dk, ik = cKDTree(P).query(P, 16)
    assert np.array_equal(ik, i1)                                   # tie-free input: exact index parity
    np.testing.assert_allclose(np.sqrt(d1), dk, rtol=1e-5, atol=1e-6)
    isk = KDTree(P).query(P[:500], 16, return_distance=False)
    assert np.array_equal(isk, i1[:500])
    # cross-set k=1 (interp_idx of randlanet.py:224)
    sub = P[:1500]
    j1, _ = O.c_knn(sub, P, 1)
    assert np.array_equal(j1[:, 0], cKDTree(sub).query(P, 1)[1])


def test_knn_batched_short_and_ties():
    P = synth.uniform_cloud(300, 2)
    P[100:110] = P[0]                      # duplicates: ties resolved by index
    ps, qs = [0, 200, 205, 300], [0, 50, 60, 100]
    Q = synth.uniform_cloud(100, 3)
    i1, d1 = O.c_knn(P, Q, 8, ps, qs)
    i2, d2 = O.np_knn(P, Q, 8, ps, qs)
    assert np.array_equal(i1, i2) and np.array_equal(d1, d2)
    assert np.all(i1[50:60, 5:] == -1) and np.all(np.isinf(d1[50:60, 5:]))   # batch item with 5 points
    assert i1[:50].max() < 200 and i1[60:].min() >= 205
    i3, _ = O.c_knn(P[:200], P[:1], 12)
    assert list(i3[0, :11]) == [0] + list(range(100, 110))


def test_radius_c_vs_numpy_vs_kdtree():
    from scipy.spatial import cKDTree
    P, _ = synth.room_cloud(5000, 5, room=(2.0, 1.6, 1.2))
    Q = P[::3]
    i1, r1, d1 = O.c_radius(P, Q, 0.1)
    i2, r2, d2 = O.np_radius(P, Q, 0.1)
    assert np.array_equal(r1, r2) and np.array_equal(i1, i2) and np.array_equal(d1, d2)
    # points on a 0.04 grid put many pairs EXACTLY at radius-like distances; compare to the
    # float64 KD-tree on a radius that is not a lattice distance
    i3, r3, _ = O.c_radius(P, Q, 0.107)
    ball = cKDTree(P).query_ball_point(Q.astype(np.float64), 0.107)
    for q in range(0, len(Q), 37):
        assert sorted(ball[q]) == sorted(i3[r3[q]:r3[q + 1]].tolist())
    # rows ascend by (d2, idx)
    for q in range(0, len(Q), 53):
        row = list(zip(d1[r1[q]:r1[q + 1]].tolist(), i1[r1[q]:r1[q + 1]].tolist()))
        assert row == sorted(row)


def test_radius_batched_empty():
    P = synth.uniform_cloud(400, 4)
    i1, r1, _ = O.c_radius(P, P[:50], 0.9, [0, 0, 400], [0, 10, 50])
    i2, r2, _ = O.np_radius(P, P[:50], 0.9, [0, 0, 400], [0, 10, 50])
    assert np.array_equal(r1, r2) and np.array_equal(i1, i2)
    assert np.all(r1[:11] == 0)             # first batch item has no support points


def test_subsample_two_restatements_agree_and_partition_the_cloud():
    """grid subsampling oracle: C (oracle_voxel_reduce) == numpy restatement bit for bit; every point
    falls in exactly one voxel; barycentres lie inside their voxel; labels are the per-voxel majority."""
    from oracle import ops as O
    rng = np.random.default_rng(3)
    pts = (rng.random((3000, 3)) * [4, 3, 2] - [1, 1, 1]).astype(np.float32)
    feats = rng.standard_normal((3000, 4)).astype(np.float32)
    labs = rng.integers(0, 5, 3000).astype(np.int32)
    lens = [1200, 0, 1800]
    a = O.c_subsample_batch(pts, lens, feats, labs, 0.25)
    b = O.np_subsample_batch(pts, lens, feats, labs, 0.25)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    sp, sl, sf, slab = a
    assert sl.sum() == len(sp) and sl[1] == 0 and len(sp) < 3000
    origin, _ = O.subsample_range(pts, 0.25)
    cell = np.floor((sp - origin) / 0.25)
    assert len(np.unique(np.concatenate([cell[:sl[0]], cell[sl[0]:] + 1000]), axis=0)) == len(sp)
    only = O.c_subsample_batch(pts, lens, None, None, 0.25)
    assert len(only) == 2 and np.array_equal(only[0], sp)
    capped = O.c_subsample_batch(pts, lens, None, None, 0.25, max_p=7)
    assert list(capped[1]) == [7, 0, 7] and np.array_equal(capped[0][:7], sp[:7])


def test_rotated_iou_oracle_known_answers():
    from oracle import ops as O
    a = np.array([[0, 0, 2, 2, 0.0]], np.float32)
    assert abs(O.c_iou_matrix(a, a, 0)[0, 0] - 1) < 1e-6
    b = np.array([[1, 0, 2, 2, 0.0], [0, 0, 2, 2, np.pi / 4], [5, 5, 1, 1, 0.3], [0, 0, 4, 1, np.pi / 2]], np.float32)
    m = O.c_iou_matrix(a, b, 0)[0]
    assert abs(m[0] - 2 / 6) < 1e-6                                   # half overlap: 2 / (4 + 4 - 2)
    oct_area = 8 * (np.sqrt(2) - 1)                                   # square x square rotated 45 deg = octagon
    assert abs(m[1] - oct_area / (8 - oct_area)) < 1e-6 and m[2] == 0
    assert abs(m[3] - 2 / 6) < 1e-6                                   # 1 x 4 upright strip crosses the square: 2
    assert np.allclose(O.c_iou_matrix(b, a, 0)[:, 0], m)              # symmetric
    rng = np.random.default_rng(1)
    for _ in range(4):
        p = np.concatenate([rng.random(2) * 2, rng.random(2) * 3 + 0.5, rng.random(1) * 6]).astype(np.float32)
        q = np.concatenate([rng.random(2) * 2, rng.random(2) * 3 + 0.5, rng.random(1) * 6]).astype(np.float32)
        iou = O.c_iou_matrix(p[None], q[None], 0)[0, 0]
        inter = iou * (p[2] * p[3] + q[2] * q[3]) / (1 + iou)
        assert abs(inter - O.np_rbox_area_mc(p.astype(np.float64), q.astype(np.float64))) < 0.05
    # 3-D: same footprint, half the height overlaps
    c = np.array([[0, 2, 0, 2, 2, 2, 0.0]], np.float32)
    d = np.array([[0, 1, 0, 2, 2, 2, 0.0]], np.float32)
    assert abs(O.c_iou_matrix(c, d, 1)[0, 0] - 4 / 12) < 1e-6


def test_nms_oracle_is_greedy_by_score():
    from oracle import ops as O
    boxes = np.array([[0, 0, 2, 2, 0], [0.1, 0, 2.1, 2, 0], [5, 5, 6, 6, 0.5], [0, 0, 2, 2, 0.05], [5, 5, 6, 6, 0.5]],
                     np.float32)
    scores = np.array([0.5, 0.9, 0.3, 0.8, 0.3], np.float32)
    keep, _ = O.c_nms(boxes, scores, 0.5)
    assert list(keep) == [1, 2]                                       # 3 and 0 overlap 1; 4 duplicates 2 (tie: 2 first)
    keep, _ = O.c_nms(boxes, scores, 0.99)
    assert list(keep) == [1, 3, 0, 2]
    assert len(O.c_nms(boxes[:0], scores[:0], 0.5)[0]) == 0


def test_sparse_conv_oracle_equals_dense_conv3d_on_a_full_lattice():
    """On a fully occupied lattice the submanifold 3x3x3 SparseConv (offset 0) is an ordinary zero-padded 3-D
    cross-correlation: checks the cell formula and the [kx, ky, kz, Cin, Cout] kernel layout against torch."""
    import torch
    from oracle import ops as O
    rng = np.random.default_rng(0)
    G, cin, cout = 5, 3, 4
    ii = np.stack(np.meshgrid(np.arange(G), np.arange(G), np.arange(G), indexing="ij"), -1).reshape(-1, 3)
    pos = (ii + 0.5).astype(np.float32)
    feat = rng.standard_normal((len(pos), cin)).astype(np.float32)
    kernel = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    got = O.c_sparse_conv(feat, pos, pos, 1.0, [0, 0, 0], kernel)
    vol = torch.from_numpy(feat).view(1, G, G, G, cin).permute(0, 4, 1, 2, 3)            # [1, C, x, y, z]
    w = torch.from_numpy(kernel).permute(4, 3, 0, 1, 2)                                  # [Cout, Cin, kx, ky, kz]
    ref = torch.nn.functional.conv3d(vol, w, padding=1).permute(0, 2, 3, 4, 1).reshape(-1, cout).numpy()
    assert np.abs(got - ref).max() < 1e-4
    # strided 2x2x2 convolution (offset -0.5) onto the coarse grid of calculate_grid (sparseconvnet.py:387-401)
    k2 = rng.standard_normal((2, 2, 2, cin, cout)).astype(np.float32)
    G2 = 4
    ii = np.stack(np.meshgrid(np.arange(G2), np.arange(G2), np.arange(G2), indexing="ij"), -1).reshape(-1, 3)
    pos = (ii + 0.5).astype(np.float32)
    feat = rng.standard_normal((len(pos), cin)).astype(np.float32)
    coarse = np.unique(ii - ii % 2, axis=0).astype(np.float32) + 0.5
    got = O.c_sparse_conv(feat, pos, coarse, 1.0, [-0.5] * 3, k2)
    vol = torch.from_numpy(feat).view(1, G2, G2, G2, cin).permute(0, 4, 1, 2, 3)
    ref = torch.nn.functional.conv3d(vol, torch.from_numpy(k2).permute(4, 3, 0, 1, 2), stride=2)
    ref = ref.permute(0, 2, 3, 4, 1).reshape(-1, cout).numpy()
    assert np.abs(got - ref).max() < 1e-4
    # transposed 2x2x2 back to the fine grid (DeConvolution: in = 2 * coarse position, sparseconvnet.py:643-646)
    cf = rng.standard_normal((len(coarse), cin)).astype(np.float32)
    up = O.c_sparse_conv(cf, coarse, pos, 1.0, [-0.5] * 3, k2, transpose=True)
    volc = torch.from_numpy(cf).view(1, 2, 2, 2, cin).permute(0, 4, 1, 2, 3)
    ref = torch.nn.functional.conv_transpose3d(volc, torch.from_numpy(k2).permute(3, 4, 0, 1, 2), stride=2)
    ref = ref.permute(0, 2, 3, 4, 1).reshape(-1, cout).numpy()
    assert np.abs(up - ref).max() < 1e-4


@pytest.mark.parametrize("v,fi,fo,transpose", [(1.0, 0.9, 0.1, False), (0.3, 0.0, 0.0, True), (0.05, 0.1, 0.8, False)])
def test_brute_force_table_contracts_to_the_sparse_conv_oracle(v, fi, fo, transpose):
    """The float32 brute-force table of the GPU table tests (tests/sparse_tables_support.py), contracted in float64,
    equals c_sparse_conv on voxel-unique inputs off the grid and at voxel corners, with bias and normalize."""
    from sparse_tables_support import brute_table, contract64
    rng = np.random.default_rng(3)
    inp = ((np.unique(rng.integers(0, 12, (900, 3)), axis=0) + 5000 + fi) * np.float32(v)).astype(np.float32)
    out = ((np.unique(rng.integers(0, 12, (400, 3)), axis=0) + 5000 + fo) * np.float32(v)).astype(np.float32)
    cin, cout = 5, 7
    feat = rng.standard_normal((len(inp), cin)).astype(np.float32)
    for ks, off in (((3, 3, 3), [0.0, 0.25, -0.25]), ((2, 3, 4), [-0.5, 0.0, -0.5])):
        kernel = rng.standard_normal(ks + (cin, cout)).astype(np.float32)
        bias = rng.standard_normal(cout).astype(np.float32)
        table, cnt = brute_table(inp, out, v, off, ks, transpose)
        assert (table < len(inp)).sum() > 1000
        for normalize in (False, True):
            want = O.c_sparse_conv(feat, inp, out, v, off, kernel, bias, normalize, transpose)
            got = contract64(feat, table, kernel)
            if normalize:
                got = got / np.maximum(cnt, 1)[:, None]
            assert np.abs(got + bias - want).max() < 1e-5 * np.abs(want).max()


def test_continuous_conv_oracle_known_answers():
    """A spatially constant filter makes the convolution a plain sum: out = (sum_n imp_n f_n) W; nearest-neighbour
    interpolation with the identity mapping on lattice offsets reproduces the sparse 3x3x3 convolution."""
    from oracle import ops as O
    rng = np.random.default_rng(2)
    n, cin, cout = 40, 3, 5
    pos = rng.random((n, 3)).astype(np.float32)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    W = rng.standard_normal((cin, cout)).astype(np.float32)
    filt = np.broadcast_to(W, (3, 3, 3, cin, cout)).copy()
    nbr = np.tile(np.arange(n), 2)
    splits = np.array([0, n, 2 * n])
    outp = np.array([[0.5, 0.5, 0.5], [0.2, 0.7, 0.1]], np.float32)
    for mapping in (0, 1):
        for interp in (0, 1):
            got = O.c_continuous_conv(filt, outp, [4.0], [0, 0, 0], pos, feat, None, nbr, None, splits, True, mapping, False, interp)
            assert np.abs(got - feat.sum(0) @ W).max() < 1e-4
    got = O.c_continuous_conv(filt, outp, [4.0], [0, 0, 0], pos, feat, None, nbr, None, splits, True, 1, True, 1)
    assert np.abs(got - feat.mean(0) @ W).max() < 1e-5
    G = 4
    ii = np.stack(np.meshgrid(np.arange(G), np.arange(G), np.arange(G), indexing="ij"), -1).reshape(-1, 3)
    lp = (ii + 0.5).astype(np.float32)
    lf = rng.standard_normal((len(lp), cin)).astype(np.float32)
    k = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)        # sparse-conv layout [x, y, z]
    ref = O.c_sparse_conv(lf, lp, lp, 1.0, [0, 0, 0], k)
    idx, rs, _ = O.c_radius(lp, lp, 1.8)                                    # the 27-neighbourhood (sqrt(3) < 1.8)
    # extent 3 voxels, align_corners: offsets {-1, 0, 1} -> p = d * 2 / 3 -> u = (p + 1) / 2 * 2 = d * 2 / 3 + 1 ... use extent 2: u = d + 1
    got = O.c_continuous_conv(np.ascontiguousarray(k.transpose(2, 1, 0, 3, 4)), lp, [2.0], [0, 0, 0], lp, lf, None, idx, None,
                              rs, True, 0, False, 0)
    assert np.abs(got - ref).max() < 1e-4


@pytest.mark.parametrize("interp", [0, 1, 2])
@pytest.mark.parametrize("align", [False, True])
def test_continuous_conv_oracle_far_neighbours_take_the_border_cell(interp, align):
    """Neighbours 1e3, 1e9 and 1e12 extents out on either side of each axis: nearest and linear take the border cell
    on that side and linear_border weighs them 0, however far out they are (a filter coordinate past 2^31 is clamped
    before it becomes an int)."""
    for sizes in ((3, 4, 5), (5, 1, 2)):
        c = far_neighbours(sizes, align, interp)
        for mapping in (0, 1):
            got = O.c_continuous_conv(c.filters, c.out_pos, [1.0], [0, 0, 0], c.inp_pos, c.feat, None, c.index, None,
                                      c.splits, align, mapping, False, interp)
            assert np.array_equal(got, c.want), (sizes, mapping, got.ravel(), c.want.ravel())
