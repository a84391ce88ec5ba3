"""Parity of the CUDA operators (through the C ABI) against the CPU oracle: bit-exact
for voxel / neighbour indices and squared distances."""
import numpy as np
import pytest
import torch

from oracle import ops as O
from open3d_ml_b200 import synth
import open3d_ml_b200 as M
from conftest import rel_err

pytestmark = pytest.mark.gpu
KITTI = dict(voxel_size=[0.16, 0.16, 4], rmin=[0, -39.68, -3], rmax=[69.12, 39.68, 1])
WAYMO = dict(voxel_size=[0.32, 0.32, 6], rmin=[-74.88, -74.88, -2], rmax=[74.88, 74.88, 4])


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def vox_check(pts, splits, g, max_pts, max_vox):
    ref = O.c_voxelize(pts[:, :3], splits, g["voxel_size"], g["rmin"], g["rmax"], max_pts, max_vox)
    rs = None if splits is None else T(np.asarray(splits, np.int64))
    out = M.voxelize(T(pts)[:, :3], rs if rs is not None else torch.tensor([0, len(pts)]).cuda(),
                     torch.tensor(g["voxel_size"]), torch.tensor(g["rmin"], dtype=torch.float32),
                     torch.tensor(g["rmax"], dtype=torch.float32), max_pts, max_vox)
    assert out.voxel_coords.dtype == torch.int32 and out.voxel_point_indices.dtype == torch.int64
    assert np.array_equal(out.voxel_coords.cpu().numpy(), ref["voxel_coords"])
    assert np.array_equal(out.voxel_point_row_splits.cpu().numpy(), ref["voxel_point_row_splits"])
    assert np.array_equal(out.voxel_point_indices.cpu().numpy(), ref["voxel_point_indices"])
    assert np.array_equal(out.voxel_batch_splits.cpu().numpy(), ref["voxel_batch_splits"])
    return ref


def test_voxelize_kitti_lidar_and_uniform():
    pts = synth.lidar_frame(20000, 3)
    pts[:7, 0] = 69.12           # p == max: kept, index == extent
    pts[7:11, 1] = 39.68
    pts[11:20, 2] = 5.0          # out of range
    pts[20:24, 0] = np.nan
    ref = vox_check(pts, None, KITTI, 32, 40000)
    assert ref["voxel_coords"][:, 0].max() == 432 and ref["voxel_coords"][:, 1].max() == 496
    vox_check(synth.uniform_frame(20000, 4), None, KITTI, 32, 40000)
    vox_check(synth.uniform_frame(20000, 4), None, KITTI, 32, 16000)     # max_voxels cap active


def test_voxelize_caps_reference_smoke_shape():
    rng = np.random.default_rng(0)      # tests/test_models.py:204-236: 10 000 pts in [0,1)^4
    pts = rng.uniform(0, 1, (10000, 4)).astype(np.float32)
    ref = vox_check(pts, None, KITTI, 32, 40000)
    assert np.diff(ref["voxel_point_row_splits"]).max() == 32
    vox_check(pts, None, KITTI, 5, 7)


def test_voxelize_batched_ragged_empty():
    frames = [synth.lidar_frame(n, 10 + i) for i, n in enumerate((5000, 0, 12345, 1))]
    pts = np.concatenate(frames)
    splits = np.concatenate([[0], np.cumsum([len(f) for f in frames])])
    vox_check(pts, splits, KITTI, 32, 3000)
    vox_check(pts, splits, KITTI, 4, 40000)
    out = M.voxelize(torch.zeros((0, 3)).cuda(), torch.tensor([0, 0]).cuda(), torch.tensor([1., 1, 1]),
                     torch.zeros(3), torch.ones(3), 4, 4)
    assert out.voxel_coords.shape == (0, 3) and out.voxel_point_row_splits.tolist() == [0]


def test_voxelize_waymo_full_size_and_3d_grid():
    vox_check(synth.lidar_frame(180000, 5, synth.WAYMO_RANGE), None, WAYMO, 20, 32000)
    g3 = dict(voxel_size=[0.5, 0.4, 0.3], rmin=[-50, -50, -3], rmax=[50, 50, 1])   # many z cells
    vox_check(synth.semantickitti_cloud(45056, 6), None, g3, 3, 100000)


def test_voxelize_is_deterministic_and_validates():
    pts = T(synth.uniform_frame(30000, 8))
    args = (torch.tensor([0, 30000]).cuda(), torch.tensor(KITTI["voxel_size"]),
            torch.tensor(KITTI["rmin"], dtype=torch.float32), torch.tensor(KITTI["rmax"], dtype=torch.float32), 32, 40000)
    a, b = M.voxelize(pts[:, :3], *args), M.voxelize(pts[:, :3], *args)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    with pytest.raises(RuntimeError):
        M.voxelize(pts[:, :2], *args)
    with pytest.raises(RuntimeError):
        M.voxelize(pts[:, :3], args[0], torch.tensor([0., 1, 1]), *args[2:])


def test_ragged_to_dense():
    rng = np.random.default_rng(1)
    lens = rng.integers(0, 40, 500)
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    v64 = rng.integers(0, 10**9, rs[-1]).astype(np.int64)
    out = M.ragged_to_dense(T(v64), T(rs), 32, torch.tensor(-1))
    assert np.array_equal(out.cpu().numpy(), O.np_ragged_to_dense(v64, rs, 32, -1))
    v32 = v64.astype(np.int32).reshape(-1, 1)          # kpconv.py:2030-2032 form: [L,1], int32 fill tensor
    out = M.ragged_to_dense(T(v32), T(rs), 36, torch.Tensor([12345]).to(torch.int32))
    assert out.shape == (500, 36, 1)
    assert np.array_equal(out.cpu().numpy(), O.np_ragged_to_dense(v32, rs, 36, np.int32(12345)))
    out = M.ragged_to_dense(torch.from_numpy(v64), torch.from_numpy(rs), 8, torch.tensor(-1))   # CPU in -> CPU out
    assert not out.is_cuda and np.array_equal(out.numpy(), O.np_ragged_to_dense(v64, rs, 8, -1))


def knn_check(P, Q, k, ps=None, qs=None, dtype=torch.int32, allow_short=False):
    ri, rd = O.c_knn(P, Q, k, ps, qs)
    r = M.knn_search(T(P), T(Q), k, None if ps is None else T(np.asarray(ps, np.int64)),
                     None if qs is None else T(np.asarray(qs, np.int64)), index_dtype=dtype,
                     return_distances=True, allow_short=allow_short)
    gi = r.neighbors_index.reshape(len(Q), k).cpu().numpy()
    gd = r.neighbors_distance.reshape(len(Q), k).cpu().numpy()
    assert gi.dtype == (np.int32 if dtype == torch.int32 else np.int64)
    assert np.array_equal(gi.astype(np.int64), ri.astype(np.int64)), "index mismatch in %d rows" % (gi != ri).any(1).sum()
    assert np.array_equal(gd, rd)
    return gi


def test_knn_small_uniform_lidar_and_cross():
    P = synth.uniform_cloud(4096, 1)                       # BASELINE config 1 shape
    knn_check(P, P, 16)
    knn_check(P[:1024], P, 1, dtype=torch.int64)           # interp_idx (randlanet.py:224)
    L_ = synth.semantickitti_cloud(8192, 2)
    knn_check(L_, L_, 16)
    knn_check(L_, synth.uniform_cloud(3000, 3, -60, 60), 5)    # queries far outside the support bbox
    knn_check(L_, L_[:100], 33)
    knn_check(L_[:2000], L_[:50], 64)


def test_knn_batched_short_items_and_duplicates():
    P = synth.uniform_cloud(3000, 4)
    P[100:110] = P[0]
    Q = synth.uniform_cloud(700, 5)
    gi = knn_check(P, Q, 8, [0, 2000, 2005, 3000], [0, 300, 350, 700], allow_short=True)
    assert (gi[300:350, 5:] == -1).all()
    with pytest.raises(RuntimeError, match="fewer than k"):        # the reference-facing op refuses ragged results
        M.knn_search(T(P), T(Q), 8, T(np.asarray([0, 2000, 2005, 3000], np.int64)), T(np.asarray([0, 300, 350, 700], np.int64)))
    knn_check(P[:2000], P[:200], 12)
    flat = synth.uniform_cloud(5000, 6)
    flat[:, 2] = 0.25                                    # degenerate (planar) extent
    knn_check(flat, flat, 16)
    same = np.repeat(synth.uniform_cloud(1, 7), 200, 0)  # all points identical: pure index order
    assert np.array_equal(knn_check(same, same, 16), np.tile(np.arange(16), (200, 1)))


def test_knn_randla_pyramid_full_size():
    """SemanticKITTI-shaped cloud, all four levels (randlanet.py:218-229), vs brute force."""
    pc = synth.semantickitti_cloud(45056, 11)
    for _ in range(4):
        gi = knn_check(pc, pc, 16)
        assert np.array_equal(gi[:, 0], np.arange(len(pc)))
        sub = pc[:len(pc) // 4]
        knn_check(sub, pc, 1, dtype=torch.int64)
        pc = sub


def test_nearest_neighbor_search_object_numpy_path():
    P = synth.uniform_cloud(2000, 8)
    nns = M.NearestNeighborSearch(M.ops._O3CTensor.from_numpy(P))
    nns.knn_index()
    idx, d = nns.knn_search(M.ops._O3CTensor.from_numpy(P[:500]), 16)
    ri, rd = O.c_knn(P, P[:500], 16)
    assert idx.numpy().dtype == np.int64 and np.array_equal(idx.numpy(), ri) and np.array_equal(d.numpy(), rd)


def radius_check(P, Q, r, ps=None, qs=None):
    ri, rrs, rd = O.c_radius(P, Q, r, ps, qs)
    out = M.fixed_radius_search(T(P), T(Q), r, None if ps is None else T(np.asarray(ps, np.int64)),
                                None if qs is None else T(np.asarray(qs, np.int64)))
    assert out.neighbors_index.dtype == torch.int32 and out.neighbors_row_splits.dtype == torch.int64
    assert np.array_equal(out.neighbors_row_splits.cpu().numpy(), rrs)
    assert np.array_equal(out.neighbors_index.cpu().numpy(), ri)
    assert np.array_equal(out.neighbors_distance.cpu().numpy(), rd)
    return rrs


def test_radius_search_room_pyramid_radii():
    P, _ = synth.room_cloud(20000, 5)
    for dl, r in ((0.04, 0.1), (0.08, 0.2), (0.16, 0.4)):
        S = P if dl == 0.04 else synth.grid_subsample(P, dl)
        radius_check(S, S, r)                                # conv neighbours
        Q = synth.grid_subsample(S, 2 * dl)
        radius_check(S, Q, r)                                # pool
        radius_check(Q, S, 2 * r)                            # upsample


def test_radius_search_batched_empty_and_layer_api():
    P = synth.uniform_cloud(3000, 9, 0, 4)
    Q = synth.uniform_cloud(500, 10, -1, 5)                  # some queries have no neighbour at all
    rrs = radius_check(P, Q, 0.3, [0, 0, 1200, 3000], [0, 40, 300, 500])
    assert (rrs[:41] == 0).all() and (np.diff(rrs) == 0).any()
    nns = M.FixedRadiusSearch()                              # kpconv.py:2021-2026, CPU tensors in/out
    res = nns(torch.from_numpy(P), torch.from_numpy(Q), 0.3, torch.tensor([0, 3000]), torch.tensor([0, 500]))
    ri, rs_, _ = O.c_radius(P, Q, 0.3)
    assert not res.neighbors_index.is_cuda and np.array_equal(res.neighbors_index.numpy(), ri)
    assert np.array_equal(res.neighbors_row_splits.numpy(), rs_)
    with pytest.raises(RuntimeError):
        M.fixed_radius_search(T(P), T(Q), -1.0)


def test_search_is_deterministic():
    P = T(synth.semantickitti_cloud(20000, 12))
    a = M.knn_search(P, P, 16, return_distances=True)
    b = M.knn_search(P, P, 16, return_distances=True)
    assert torch.equal(a.neighbors_index, b.neighbors_index) and torch.equal(a.neighbors_distance, b.neighbors_distance)
    c, d = M.fixed_radius_search(P, P, 0.5), M.fixed_radius_search(P, P, 0.5)
    assert torch.equal(c.neighbors_index, d.neighbors_index) and torch.equal(c.neighbors_row_splits, d.neighbors_row_splits)


# ------------------------------------------------------------------ grid subsampling (f1)
@pytest.mark.parametrize("dl,lens", [(0.25, [1200, 0, 1800]), (0.04, [20000]), (1.5, [500, 500])])
def test_subsample_batch_bit_exact_vs_oracle(dl, lens):
    import open3d_ml_b200 as M
    from oracle import ops as O
    rng = np.random.default_rng(5)
    n = sum(lens)
    pts = (rng.random((n, 3)) * [4, 3, 2] - [1, 1, 1]).astype(np.float32)
    feats = rng.standard_normal((n, 5)).astype(np.float32)
    labs = rng.integers(0, 6, n).astype(np.int64)
    got = M.subsample_batch(pts, lens, features=feats, classes=labs, sampleDl=dl)
    ref = O.c_subsample_batch(pts, lens, feats, labs, dl)
    assert len(got) == 4 and got[3].dtype == np.int64
    for g, r in zip(got, ref):
        assert np.array_equal(np.asarray(g).astype(r.dtype), r)
    g2 = M.subsample_batch(pts, lens, sampleDl=dl, max_p=9)
    r2 = O.c_subsample_batch(pts, lens, None, None, dl, max_p=9)
    assert len(g2) == 2 and np.array_equal(g2[0], r2[0]) and np.array_equal(g2[1], r2[1])


def test_subsample_single_cloud_signatures():
    """The four call shapes of DataProcessing.grid_subsampling (dataprocessing.py:33-49)."""
    import open3d_ml_b200 as M
    from oracle import ops as O
    rng = np.random.default_rng(6)
    pts = rng.random((5000, 3)).astype(np.float32) * 3
    feats = rng.random((5000, 3)).astype(np.float32)
    labs = rng.integers(0, 4, 5000).astype(np.int32)
    ref = O.c_subsample_batch(pts, [5000], feats, labs, 0.2)
    p = M.subsample(pts, sampleDl=0.2)
    assert isinstance(p, np.ndarray) and np.array_equal(p, ref[0])
    p, f = M.subsample(pts, features=feats, sampleDl=0.2)
    assert np.array_equal(p, ref[0]) and np.array_equal(f, ref[2])
    p, l = M.subsample(pts, classes=labs, sampleDl=0.2)
    assert np.array_equal(l, ref[3])
    p, f, l = M.subsample(pts, features=feats, classes=labs, sampleDl=0.2)
    assert np.array_equal(f, ref[2]) and np.array_equal(l, ref[3])


# ------------------------------------------------------------------ rotated IoU / NMS (f2)
def _rand_boxes(n, seed, spread=20.0):
    rng = np.random.default_rng(seed)
    c = rng.random((n, 2)) * spread
    wh = rng.random((n, 2)) * 3 + 0.5
    r = (rng.random((n, 1)) - 0.5) * 2 * np.pi
    return np.concatenate([c, wh, r], 1).astype(np.float32)


@pytest.mark.parametrize("na,nb", [(1, 1), (37, 53), (300, 200)])
def test_iou_bev_and_3d_vs_oracle(na, nb):
    import open3d_ml_b200 as M
    from oracle import ops as O
    a, b = _rand_boxes(na, 1, 8.0), _rand_boxes(nb, 2, 8.0)
    got = M.iou_bev(a, b)
    assert isinstance(got, np.ndarray) and np.abs(got - O.c_iou_matrix(a, b, 0)).max() < 2e-5
    rng = np.random.default_rng(3)
    def to3d(x, seed):
        y = rng.random((len(x), 1)) * 2
        h = rng.random((len(x), 1)) * 2 + 0.5
        return np.concatenate([x[:, :1], y, x[:, 1:2], x[:, 2:3], h, x[:, 3:4], x[:, 4:5]], 1).astype(np.float32)
    a3, b3 = to3d(a, 4), to3d(b, 5)
    got3 = M.iou_3d(torch.from_numpy(a3).cuda(), torch.from_numpy(b3).cuda())
    assert got3.is_cuda and np.abs(got3.cpu().numpy() - O.c_iou_matrix(a3, b3, 1)).max() < 2e-5
    assert M.iou_bev(a[:0], b).shape == (0, nb)


@pytest.mark.parametrize("n,thr,spread", [(1, 0.5, 5.0), (100, 0.01, 20.0), (1000, 0.32, 30.0), (4097, 0.5, 60.0), (513, 0.01, 3.0)])
def test_nms_vs_oracle(n, thr, spread):
    """Kept indices equal the oracle's whenever no decisive IoU lies within fp32 noise of the threshold
    (the oracle reports the closest approach; the seeds here keep it above 1e-5)."""
    import open3d_ml_b200 as M
    from oracle import ops as O
    bx = _rand_boxes(n, 7 + n, spread)
    boxes = np.stack([bx[:, 0] - bx[:, 2] / 2, bx[:, 1] - bx[:, 3] / 2, bx[:, 0] + bx[:, 2] / 2, bx[:, 1] + bx[:, 3] / 2,
                      bx[:, 4]], 1).astype(np.float32)
    scores = np.random.default_rng(n).random(n).astype(np.float32)
    scores[n // 2:] = scores[:n - n // 2]                    # exact ties: lower index first
    ref, gap = O.c_nms(boxes, scores, thr)
    assert gap > 1e-5 or n == 1
    got = M.nms(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), thr)
    assert got.dtype == torch.int64 and got.is_cuda and np.array_equal(got.cpu().numpy(), ref)
    got_cpu = M.nms(torch.from_numpy(boxes), torch.from_numpy(scores), thr)
    assert not got_cpu.is_cuda and np.array_equal(got_cpu.numpy(), ref)


def test_nms_empty_and_bad_shapes():
    import open3d_ml_b200 as M
    assert M.nms(torch.zeros(0, 5).cuda(), torch.zeros(0).cuda(), 0.5).numel() == 0
    with pytest.raises(RuntimeError):
        M.nms(torch.zeros(4, 4).cuda(), torch.zeros(4).cuda(), 0.5)


# ------------------------------------------------------------------ SparseConvUnet ops (f3) + voxel_pooling (f4)
def _sparse_lattice(n_vox, grid, seed):
    rng = np.random.default_rng(seed)
    ii = np.unique(rng.integers(0, grid, (n_vox, 3)), axis=0)
    return ii.astype(np.int64)


@pytest.mark.parametrize("cin,cout,normalize,bias", [(32, 64, False, False), (64, 32, True, True), (5, 7, False, True)])
def test_sparse_conv_layers_vs_oracle(cin, cout, normalize, bias):
    """SubmanifoldSparseConv (3^3, offset 0), Convolution (2^3, offset -0.5, onto calculate_grid's coarse lattice)
    and DeConvolution (transposed 2^3) of sparseconvnet.py:344-485 against the brute-force oracle, whose cell
    formula is itself pinned to torch conv3d / conv_transpose3d (tests/test_oracle_ops.py)."""
    from open3d_ml_b200 import layers as LY
    from oracle import ops as O
    ii = _sparse_lattice(3000, 24, 11)
    pos = (ii + 0.5).astype(np.float32)
    rng = np.random.default_rng(12)
    feat = rng.standard_normal((len(pos), cin)).astype(np.float32)
    torch.manual_seed(0)
    with torch.no_grad():
        # submanifold
        conv = LY.SparseConv(cin, cout, [3, 3, 3], use_bias=bias, normalize=normalize, offset=torch.zeros(3)).eval()
        if bias:
            conv.bias.normal_()
        got = conv(torch.from_numpy(feat), torch.from_numpy(pos), torch.from_numpy(pos), 1.0)
        ref = O.c_sparse_conv(feat, pos, pos, 1.0, [0, 0, 0], conv.kernel.numpy(), conv.bias.numpy() if bias else None,
                              normalize)
        assert not got.is_cuda and rel_err(got, ref) < 1e-4
        # strided down
        coarse = (np.unique(ii - ii % 2, axis=0) + 0.5).astype(np.float32)
        down = LY.SparseConv(cin, cout, [2, 2, 2], use_bias=bias, normalize=normalize, offset=torch.full((3,), -0.5)).eval()
        got = down(torch.from_numpy(feat).cuda(), torch.from_numpy(pos).cuda(), torch.from_numpy(coarse).cuda(), 1.0)
        ref = O.c_sparse_conv(feat, pos, coarse, 1.0, [-0.5] * 3, down.kernel.numpy(), down.bias.numpy() if bias else None,
                              normalize)
        assert got.is_cuda and rel_err(got, ref) < 1e-4
        # transposed up
        cf = rng.standard_normal((len(coarse), cin)).astype(np.float32)
        up = LY.SparseConvTranspose(cin, cout, [2, 2, 2], use_bias=bias, normalize=normalize, offset=torch.full((3,), -0.5)).eval()
        got = up(torch.from_numpy(cf), torch.from_numpy(coarse), torch.from_numpy(pos), 1.0)
        ref = O.c_sparse_conv(cf, coarse, pos, 1.0, [-0.5] * 3, up.kernel.numpy(), up.bias.numpy() if bias else None,
                              normalize, transpose=True)
        assert rel_err(got, ref) < 1e-4
        # state_dict keys are the upstream layer's
        assert set(k for k in conv.state_dict() if k != "offset") == ({"kernel", "bias"} if bias else {"kernel"})


def test_reduce_subarrays_sum_and_voxel_pooling():
    import open3d_ml_b200 as M
    from oracle import ops as O
    rng = np.random.default_rng(13)
    vals = rng.standard_normal(5000).astype(np.float32)
    rs = np.concatenate([[0], np.sort(rng.integers(0, 5000, 300)), [5000]]).astype(np.int64)
    got = M.ops.reduce_subarrays_sum(torch.from_numpy(vals).cuda(), torch.from_numpy(rs).cuda())
    assert np.array_equal(got.cpu().numpy(), O.c_reduce_subarrays_sum(vals, rs))
    pts = (rng.random((4000, 3)) * 3).astype(np.float32)
    feats = rng.standard_normal((4000, 6)).astype(np.float32)
    r = M.ops.voxel_pooling(torch.from_numpy(pts).cuda(), torch.from_numpy(feats).cuda(), 0.5, "average", "max")
    vox = np.floor(pts / 0.5).astype(np.int64)
    keys = vox[:, 0] + 100 * (vox[:, 1] + 100 * vox[:, 2])
    uk = np.unique(keys)
    assert r.pooled_positions.shape == (len(uk), 3) and r.pooled_features.shape == (len(uk), 6)
    order = np.argsort(keys, kind="stable")
    ks = keys[order]
    first = np.searchsorted(ks, uk)
    last = np.searchsorted(ks, uk, side="right")
    ref_f = np.stack([feats[order[a:b]].max(0) for a, b in zip(first, last)])
    ref_p = np.stack([pts[order[a:b]].astype(np.float64).mean(0) for a, b in zip(first, last)])
    assert np.array_equal(r.pooled_features.cpu().numpy(), ref_f)
    assert np.abs(r.pooled_positions.cpu().numpy() - ref_p).max() < 1e-5
    c = M.ops.voxel_pooling(torch.from_numpy(pts), torch.from_numpy(feats), 0.5, "center", "nearest_neighbor")
    assert not c.pooled_positions.is_cuda
    assert np.allclose(c.pooled_positions.numpy(), (np.floor(ref_p / 0.5) + 0.5) * 0.5)
    d2 = ((pts - (np.floor(pts / 0.5) + 0.5) * 0.5) ** 2).sum(1)
    nn = np.array([order[a:b][np.argmin(d2[order[a:b]])] for a, b in zip(first, last)])
    assert np.array_equal(c.pooled_features.numpy(), feats[nn])


def test_raw_sparse_conv_op_vs_dense_table():
    import open3d_ml_b200 as M
    from oracle import ops as O
    ii = _sparse_lattice(800, 12, 31)
    pos = (ii + 0.5).astype(np.float32)
    rng = np.random.default_rng(32)
    cin, cout = 32, 16
    feat = rng.standard_normal((len(pos), cin)).astype(np.float32)
    k = rng.standard_normal((3, 3, 3, cin, cout)).astype(np.float32)
    ref = O.c_sparse_conv(feat, pos, pos, 1.0, [0, 0, 0], k)
    # ragged neighbour lists (index, kernel cell) of the 27-neighbourhood, built on the host
    key = {tuple(v): i for i, v in enumerate(ii)}
    nidx, kidx, rs = [], [], [0]
    for v in ii:
        for dx in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dz in (-1, 0, 1):
                    j = key.get((v[0] + dx, v[1] + dy, v[2] + dz))
                    if j is not None:
                        nidx.append(j)
                        kidx.append(((dx + 1) * 3 + (dy + 1)) * 3 + (dz + 1))
        rs.append(len(nidx))
    got = M.ops.sparse_conv(torch.from_numpy(k), torch.from_numpy(feat).cuda(), torch.empty(0),
                            torch.tensor(nidx, dtype=torch.int32).cuda(), torch.tensor(kidx, dtype=torch.uint8).cuda(),
                            torch.empty(0), torch.tensor(rs, dtype=torch.int64).cuda())
    assert rel_err(got, ref) < 1e-4
