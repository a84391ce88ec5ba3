"""The general neighbour searches on the GPU: radius_search (one radius per query), the L1 / Linf metrics,
ignore_query_point, normalize_distances and index_dtype of fixed_radius_search / radius_search / knn_search, bit-equal
to the oracle (oracle/search.py c_search_*) on uniform, LiDAR-like and room clouds; the layers from CPU and CUDA tensors
and through the shim; repeatability; launch counts against a profiler trace (in a process of its own); exact
workspaces; layers.ContinuousConv with the new search options, window and user lists; and the adjoint identity of
ContinuousConvTranspose with an L1 search that ignores query points."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import open3d_ml_b200 as M
from open3d_ml_b200 import _lib as L, layers as LY, synth
from oracle import ops as O, search as S
from conftest import ROOT, rel_err
from test_gpu_launch_count import counted_and_traced

pytestmark = pytest.mark.gpu

METRICS = ["L2", "L1", "Linf"]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def room(n, seed):
    r = synth.room_cloud(n, seed)
    return np.ascontiguousarray(r[0] if isinstance(r, tuple) else r, np.float32)


def batch_case(kind, seed=0):
    """(points, queries, point splits, query splits, scalar radius): three batch items, the middle one without points
    (its queries get empty rows) plus one item without queries; queries partly outside the support box, some on support
    points, and coincident duplicates among the points."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        mk, radius = (lambda n, s: synth.uniform_cloud(n, s, 0.0, 1.0)), 0.08
    elif kind == "lidar":
        mk, radius = (lambda n, s: synth.semantickitti_cloud(n, s)), 1.0
    else:
        mk, radius = room, 0.1
    a, b, c = mk(3000, seed), mk(2500, seed + 1), mk(200, seed + 2)
    a[10:20] = a[0]
    pts = np.concatenate([a, b, c]).astype(np.float32)
    ps = np.array([0, 3000, 3000, 5500, 5700], np.int64)
    lo, hi = pts.min(0), pts.max(0)
    qa = rng.uniform(lo - 0.1 * (hi - lo), hi + 0.1 * (hi - lo), (700, 3)).astype(np.float32)
    qa[::3] = a[rng.integers(0, 3000, len(qa[::3]))]
    qa[1] = a[0]
    qb = rng.uniform(lo, hi, (50, 3)).astype(np.float32)
    qc = b[rng.integers(0, 2500, 400)]
    q = np.concatenate([qa, qb, qc]).astype(np.float32)
    qs = np.array([0, 700, 750, 1150, 1150], np.int64)
    return pts, q, ps, qs, radius


def radii_for(rng, q, radius):
    r = (rng.uniform(0.3, 3.0, len(q)) * radius).astype(np.float32)     # a 10x spread
    r[1], r[2], r[4], r[5], r[7] = 0, -radius, np.nan, np.inf, -0.0
    return r


def check_radius(res, ref, index_dtype, want_dist):
    idx, rs, d = ref
    assert res.neighbors_index.dtype == index_dtype and res.neighbors_index.is_cuda
    assert np.array_equal(res.neighbors_row_splits.cpu().numpy(), rs)
    assert np.array_equal(res.neighbors_index.cpu().numpy().astype(np.int64), idx)
    if want_dist:
        assert np.array_equal(res.neighbors_distance.cpu().numpy(), d, equal_nan=True)
    else:
        assert res.neighbors_distance.numel() == 0


@pytest.mark.parametrize("kind", ["uniform", "lidar", "room"])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_fixed_radius_search_bit_equal_to_oracle(kind, metric, ignore):
    pts, q, ps, qs, radius = batch_case(kind)
    for index_dtype in (torch.int32, torch.int64):
        res = M.ops.fixed_radius_search(T(pts), T(q), radius, T(ps), T(qs), index_dtype=index_dtype, metric=metric,
                                        ignore_query_point=ignore)
        ref = S.c_search_radius(pts, q, radius, None, ps, qs, S.METRICS[metric], ignore)
        assert ref[1][-1] > 0
        check_radius(res, ref, index_dtype, True)


@pytest.mark.parametrize("kind", ["uniform", "lidar", "room"])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore,normalize", [(False, False), (True, True), (False, True)])
def test_radius_search_bit_equal_to_oracle(kind, metric, ignore, normalize):
    pts, q, ps, qs, radius = batch_case(kind, seed=1)
    radii = radii_for(np.random.default_rng(2), q, radius)
    for index_dtype in (torch.int32, torch.int64):
        res = M.ops.radius_search(T(pts), T(q), T(radii), T(ps), T(qs), index_dtype=index_dtype, metric=metric,
                                  ignore_query_point=ignore, return_distances=True,
                                  normalize_distances=normalize)
        ref = S.c_search_radius(pts, q, 0.0, radii, ps, qs, S.METRICS[metric], ignore, normalize)
        check_radius(res, ref, index_dtype, True)
    lens = np.diff(ref[1])
    assert lens[2] == lens[4] == lens[5] == 0 and lens[1] == (0 if ignore else 11)


def test_radius_search_with_constant_radii_equals_fixed_radius_search():
    pts, q, ps, qs, radius = batch_case("room", seed=3)
    radii = torch.full((len(q),), radius, dtype=torch.float32).cuda()
    for metric in METRICS:
        a = M.ops.fixed_radius_search(T(pts), T(q), radius, T(ps), T(qs), metric=metric)
        b = M.ops.radius_search(T(pts), T(q), radii, T(ps), T(qs), metric=metric, return_distances=True)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_item_whose_radii_are_all_invalid_or_zero():
    rng = np.random.default_rng(4)
    pts = rng.uniform(0, 100, (500, 3)).astype(np.float32)     # a large box: the 1e-6 cell floor must still fit
    q = np.concatenate([pts[:5], rng.uniform(0, 100, (5, 3))]).astype(np.float32)
    for radii in (np.zeros(10, np.float32), np.full(10, np.nan, np.float32), np.full(10, 1e-7, np.float32)):
        res = M.ops.radius_search(T(pts), T(q), T(radii), return_distances=True)
        check_radius(res, S.c_search_radius(pts, q, 0.0, radii), torch.int32, True)
    res = M.ops.fixed_radius_search(T(pts), T(q), 1e-6)          # the same floor in the scalar search
    check_radius(res, S.c_search_radius(pts, q, 1e-6), torch.int32, True)
    res = M.ops.fixed_radius_search(T(pts), T(pts[:3] + 200), 1.0)   # no neighbour at all: empty rows
    assert res.neighbors_index.numel() == 0 and res.neighbors_row_splits.tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("kind", ["uniform", "lidar", "room"])
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
@pytest.mark.parametrize("k", [1, 5, 16, 33])
def test_knn_search_bit_equal_to_oracle(kind, metric, ignore, k):
    pts, q, ps, qs, _ = batch_case(kind, seed=5)
    ps = np.array([0, 3000, 3100, 5500, 5700], np.int64)       # every item holds at least k points
    pts[3000:3080] = q[700]                                     # 80 of item 1's 100 points on its first query
    ref_idx, ref_d, ref_n = S.c_search_knn(pts, q, k, ps, qs, S.METRICS[metric], ignore)
    for index_dtype in (torch.int32, torch.int64):
        res = M.ops.knn_search(T(pts), T(q), k, T(ps), T(qs), index_dtype=index_dtype, metric=metric,
                               ignore_query_point=ignore, return_distances=True)
        assert res.neighbors_index.dtype == index_dtype
        rs = np.concatenate([[0], np.cumsum(ref_n)])
        assert np.array_equal(res.neighbors_row_splits.cpu().numpy(), rs)
        keep = np.arange(k)[None, :] < ref_n[:, None]
        assert np.array_equal(res.neighbors_index.cpu().numpy().astype(np.int64), ref_idx[keep])
        assert np.array_equal(res.neighbors_distance.cpu().numpy(), ref_d[keep])
    short = ignore and k > 20                                   # query 700 keeps 20 points when it ignores the 80
    assert ref_n[700] == (20 if short else k)
    assert (np.delete(ref_n, 700) == k).all()


def test_layers_cpu_and_cuda_and_shim():
    pts, q, ps, qs, radius = batch_case("uniform", seed=6)
    radii = np.full(len(q), radius, np.float32)
    layers = [(M.ops.FixedRadiusSearch(metric="L1", ignore_query_point=True, return_distances=True,
                                       index_dtype=torch.int64), (radius,)),
              (M.ops.RadiusSearch(metric="Linf", ignore_query_point=True, return_distances=True,
                                  normalize_distances=True, index_dtype=torch.int64), (radii,)),
              (M.ops.KNNSearch(metric="L1", ignore_query_point=True, return_distances=True, index_dtype=torch.int64),
               (8,))]
    for layer, (arg,) in layers:
        sp = ps if not isinstance(layer, M.ops.KNNSearch) else np.array([0, 3000, 3100, 5500, 5700], np.int64)
        cpu = layer(torch.from_numpy(pts), torch.from_numpy(q),
                    torch.from_numpy(arg) if isinstance(arg, np.ndarray) else arg,
                    torch.from_numpy(sp), torch.from_numpy(qs))
        gpu = layer(T(pts), T(q), T(arg) if isinstance(arg, np.ndarray) else arg, T(sp), T(qs))
        assert not any(t.is_cuda for t in cpu) and all(t.is_cuda for t in gpu)
        assert cpu.neighbors_index.dtype == torch.int64
        for a, b in zip(cpu, gpu):
            assert torch.equal(a, b.cpu())
    ref = S.c_search_radius(pts, q, 0.0, radii, ps, qs, 2, True, True)
    assert np.array_equal(layers[1][0](T(pts), T(q), T(radii), T(ps), T(qs)).neighbors_distance.cpu().numpy(), ref[2])
    code = ("import open3d_ml_b200.shim as s; s.install(); import open3d.ml.torch as ml3d; "
            "print(ml3d.ops.radius_search.__name__, ml3d.layers.RadiusSearch.__name__)")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.split() == ["radius_search", "RadiusSearch"], r.stderr[-2000:]


def test_refusals():
    p = torch.rand(20, 3).cuda()
    with pytest.raises(RuntimeError, match="metric"):
        M.ops.fixed_radius_search(p, p, 0.1, metric="L3")
    with pytest.raises(RuntimeError, match="metric"):
        M.ops.KNNSearch(metric="cosine")
    with pytest.raises(RuntimeError, match="index_dtype"):
        M.ops.radius_search(p, p, torch.full((20,), 0.1).cuda(), index_dtype=torch.int16)
    with pytest.raises(RuntimeError, match="one radius per query"):
        M.ops.radius_search(p, p, torch.full((19,), 0.1).cuda())
    with pytest.raises(RuntimeError, match="positive"):
        M.ops.fixed_radius_search(p, p, 0.0, metric="L1")
    with pytest.raises(RuntimeError, match="fewer than k"):
        M.ops.knn_search(p, p, 21, ignore_query_point=True)


def test_runs_repeat_bit_for_bit():
    pts, q, ps, qs, radius = batch_case("lidar", seed=7)
    radii = T(radii_for(np.random.default_rng(8), q, radius))

    def run():
        a = M.ops.radius_search(T(pts), T(q), radii, T(ps), T(qs), metric="L1", ignore_query_point=True,
                                return_distances=True, normalize_distances=True)
        b = M.ops.knn_search(T(pts), T(q), 9, T(ps), T(qs), metric="Linf", ignore_query_point=True,
                             return_distances=True, allow_short=True)
        return list(a) + list(b)
    first = run()
    for _ in range(3):
        for x, y in zip(first, run()):
            assert torch.equal(x, y) or (x.dtype.is_floating_point and torch.equal(x.isnan(), y.isnan()) and
                                         torch.equal(x.nan_to_num(), y.nan_to_num()))


# ------------------------------------------------------------------------------------------------ the C ABI
class SearchCase:
    """One o3dml_radius_search_count + _fill (radii given) or one o3dml_knn_search_metric call, inputs on the GPU."""

    def __init__(self, what, num_points=2000, num_queries=900, batch_splits=((0, 1200, 2000), (0, 500, 900))):
        rng = np.random.default_rng(9)
        self.what = what
        self.p = T(rng.random((num_points, 3)).astype(np.float32))
        self.q = T(rng.random((num_queries, 3)).astype(np.float32))
        self.ps, self.qs = T(np.array(batch_splits[0], np.int64)), T(np.array(batch_splits[1], np.int64))
        self.np, self.nq, self.batch = num_points, num_queries, len(batch_splits[0]) - 1
        self.radii = T(rng.uniform(0.02, 0.08, num_queries).astype(np.float32))
        self.rs = torch.empty(num_queries + 1, dtype=torch.int64).cuda()
        self.total = torch.zeros(1, dtype=torch.int64).cuda()
        self.k = 12
        if what == "knn":
            self.wsb = L.lib().o3dml_knn_search_metric_workspace_bytes(num_points, num_queries, self.batch, self.k, 1)
            self.idx = torch.empty(num_queries * self.k, dtype=torch.int64).cuda()
            self.d = torch.empty(num_queries * self.k).cuda()
        else:
            self.wsb = L.lib().o3dml_radius_workspace_bytes(num_points, num_queries, self.batch)

    def count(self, ws, nbytes):
        if self.what == "knn":
            return L.lib().o3dml_knn_search_metric(L.ptr(self.p), self.np, L.ptr(self.ps), L.ptr(self.q), self.nq,
                                                   L.ptr(self.qs), self.batch, self.k, 1, 1, L.ptr(self.idx), 1,
                                                   L.ptr(self.d), L.ptr(self.rs), L.ptr(self.total), ws, nbytes,
                                                   L.stream())
        return L.lib().o3dml_radius_search_count(L.ptr(self.p), self.np, L.ptr(self.ps), L.ptr(self.q), self.nq,
                                                 L.ptr(self.qs), self.batch, 0.0, L.ptr(self.radii), 2, 1,
                                                 L.ptr(self.rs), L.ptr(self.total), ws, nbytes, L.stream())

    def prepare_fill(self):
        t = int(self.total.item())
        self.idx, self.d = torch.zeros(t, dtype=torch.int64).cuda(), torch.zeros(t).cuda()

    def fill(self, ws, nbytes):
        return L.lib().o3dml_radius_search_fill(L.ptr(self.q), self.np, self.nq, L.ptr(self.qs), self.batch, 0.0,
                                                L.ptr(self.radii), 2, 1, 1, L.ptr(self.rs), L.ptr(self.idx), 1,
                                                L.ptr(self.d), ws, nbytes, L.stream())

    def reference(self):
        p, q = self.p.cpu().numpy(), self.q.cpu().numpy()
        ps, qs = self.ps.cpu().numpy(), self.qs.cpu().numpy()
        if self.what == "knn":
            idx, d, n = S.c_search_knn(p, q, self.k, ps, qs, 1, True)
            keep = np.arange(self.k)[None, :] < n[:, None]
            return idx[keep], np.concatenate([[0], np.cumsum(n)]), d[keep]
        return S.c_search_radius(p, q, 0.0, self.radii.cpu().numpy(), ps, qs, 2, True, True)


def launch_call(what):
    case = SearchCase(what)
    ws = torch.empty(case.wsb, dtype=torch.uint8).cuda()
    if what == "radius_fill":
        L.check(case.count(L.ptr(ws), case.wsb))
        case.prepare_fill()
        return lambda: case.fill(L.ptr(ws), case.wsb)
    return lambda: case.count(L.ptr(ws), case.wsb)


LAUNCH_CASES = {
    "radius_search_count": lambda: launch_call("radius_count"),
    "radius_search_fill": lambda: launch_call("radius_fill"),
    "knn_search_metric_ignore": lambda: launch_call("knn"),
}
EXPECT = {"radius_search_count": "radius_kernel<0,2,true,true>", "radius_search_fill": "radius_kernel<1,2,true,true>",
          "knn_search_metric_ignore": "knn_compact_kernel"}


def profile_launch_cases():
    out = {}
    for case, build in LAUNCH_CASES.items():
        call = build()
        for _ in range(3):      # a session now and then delivers no records at all (see test_gpu_launch_count)
            counted, names = counted_and_traced(call)
            if names:
                break
        out[case] = (counted, names)
    return out


@pytest.fixture(scope="module")
def launch_profiles():
    """profile_launch_cases in a process of its own, for the reason given in test_gpu_cconv_transpose.py."""
    code = "import json, test_gpu_search as t; print(json.dumps(t.profile_launch_cases()))"
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", list(LAUNCH_CASES))
def test_launch_count_matches_profiled_kernels(case, launch_profiles):
    counted, names = launch_profiles[case]
    assert names and counted == len(names), (case, counted, names)
    assert any(EXPECT[case] in n.replace(" ", "") for n in names), names


TAIL, PATTERN = 4096, 0xA5


@pytest.mark.parametrize("what", ["radius", "knn"])
def test_exact_workspace_suffices_and_one_byte_less_is_refused(what):
    case = SearchCase(what)
    wsb = case.wsb
    buf = torch.full((wsb + TAIL,), PATTERN, dtype=torch.uint8, device="cuda")
    L.check(case.count(L.ptr(buf), wsb))
    if what == "radius":
        case.prepare_fill()
        L.check(case.fill(L.ptr(buf), wsb))
    torch.cuda.synchronize()
    ref_idx, ref_rs, ref_d = case.reference()
    t = int(case.total.item())
    assert np.array_equal(case.rs.cpu().numpy(), ref_rs) and t == ref_rs[-1]
    assert np.array_equal(case.idx[:t].cpu().numpy(), ref_idx)
    assert np.array_equal(case.d[:t].cpu().numpy(), ref_d)
    assert bool((buf[wsb:] == PATTERN).all()), "wrote past its %d-byte workspace" % wsb
    calls = [case.count] + ([case.fill] if what == "radius" else [])
    for call in calls:
        n0 = L.lib().o3dml_launch_count()
        assert call(L.ptr(buf), wsb - 1) == 2, L.lib().o3dml_last_error().decode()
        assert ("(%d needed)" % wsb) in L.lib().o3dml_last_error().decode()
        assert L.lib().o3dml_launch_count() == n0


# ------------------------------------------------------------------------------------------- ContinuousConv
def poly6(r2):
    return torch.clamp((1 - r2) ** 3, 0, 1)


def conv_case(seed=10, n=400, m=300, cin=5, cout=6):
    rng = np.random.default_rng(seed)
    ip = rng.random((n, 3)).astype(np.float32)
    op = np.concatenate([ip[:60], rng.random((m - 60, 3))]).astype(np.float32)   # outputs on inputs
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    return ip, op, feat, cin, cout


def oracle_conv(layer, ip, op, feat, ext, idx, rs, imp):
    return O.c_continuous_conv(layer.kernel.detach().numpy(), op, ext, layer.offset.numpy(), ip, feat, None, idx, imp,
                               rs, layer.align_corners, 1, layer.normalize, 1) + layer.bias.detach().numpy()


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
@pytest.mark.parametrize("per_point", [False, True])
@pytest.mark.parametrize("window", [False, True])
def test_continuous_conv_layer_search_options(metric, ignore, per_point, window):
    ip, op, feat, cin, cout = conv_case()
    rng = np.random.default_rng(11)
    ext = (rng.uniform(0.15, 0.4, len(op)) if per_point else np.array([0.3])).astype(np.float32)
    with torch.no_grad():
        layer = LY.ContinuousConv(cin, cout, [3, 3, 3], radius_search_metric=metric,
                                  radius_search_ignore_query_points=ignore,
                                  window_function=poly6 if window else None).eval()
        layer.bias.normal_()
        got = layer(torch.from_numpy(feat), torch.from_numpy(ip), torch.from_numpy(op), torch.from_numpy(ext))
    m = S.METRICS[metric]
    if per_point:
        idx, rs, d = S.c_search_radius(ip, op, 0.0, ext * np.float32(0.5), None, None, m, ignore, True)
    else:
        r = np.float32(ext[0] * np.float32(0.5))
        idx, rs, d = S.c_search_radius(ip, op, float(r), None, None, None, m, ignore, False)
        d = d / (np.float32(r * r) if m == 0 else r)
    imp = poly6(torch.from_numpy(d.astype(np.float32))).numpy() if window else None
    want = oracle_conv(layer, ip, op, feat, ext, idx, rs, imp)
    assert rel_err(got, want) < 1e-4


def test_continuous_conv_layer_user_neighbors():
    ip, op, feat, cin, cout = conv_case(12)
    rng = np.random.default_rng(13)
    lens = rng.integers(0, 6, len(op))
    rs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(0, len(ip), rs[-1]).astype(np.int64)
    imp = rng.random(rs[-1]).astype(np.float32)
    with torch.no_grad():
        layer = LY.ContinuousConv(cin, cout, [4, 4, 4], window_function=poly6).eval()
        layer.bias.normal_()
        got = layer(T(feat), T(ip), T(op), 0.3, user_neighbors_index=T(idx), user_neighbors_row_splits=T(rs),
                    user_neighbors_importance=T(imp))
    want = oracle_conv(layer, ip, op, feat, [0.3], idx, rs, imp)
    assert got.is_cuda and rel_err(got, want) < 1e-4


def test_continuous_conv_use_dense_layer_for_center_refused():
    with pytest.raises(RuntimeError, match="use_dense_layer_for_center"):
        LY.ContinuousConv(3, 4, [3, 3, 3], use_dense_layer_for_center=True)


def test_transpose_adjoint_with_l1_search_ignoring_query_points():
    rng = np.random.default_rng(14)
    n, m, cin, cout, ext = 400, 900, 8, 5, 0.35
    ipn = rng.random((n, 3)).astype(np.float32)
    opn = np.concatenate([ipn[:100], rng.random((m - 100, 3))]).astype(np.float32)
    ip, op = T(ipn), T(opn)
    x, y = T(rng.standard_normal((n, cin)).astype(np.float32)), T(rng.standard_normal((m, cout)).astype(np.float32))
    kw = dict(align_corners=True, coordinate_mapping="ball_to_cube_radial", interpolation="linear", normalize=False,
              use_bias=False, radius_search_metric="L1", radius_search_ignore_query_points=True)
    with torch.no_grad():
        t = LY.ContinuousConvTranspose(cin, cout, [4, 4, 4], **kw).eval()
        f = LY.ContinuousConv(cout, cin, [4, 4, 4], **kw).eval()
        f.kernel.copy_(t.kernel.transpose(-1, -2))
        tx = t(x, ip, op, ext)
        fy = f(y, op, ip, ext)
    a, b = (fy.double() * x.double()).sum(), (y.double() * tx.double()).sum()
    terms = (fy.double() * x.double()).abs().sum() + (y.double() * tx.double()).abs().sum()
    assert float(terms) > 0 and float((a - b).abs()) <= 1e-4 * float(terms)
    # the search really skipped the coincident pairs: with them the result differs
    kw["radius_search_ignore_query_points"] = False
    with torch.no_grad():
        t2 = LY.ContinuousConvTranspose(cin, cout, [4, 4, 4], **kw).eval()
        t2.kernel.copy_(t.kernel)
        assert not torch.equal(t2(x, ip, op, ext), tx)
