"""The gathered GEMM / implicit-GEMM conv / pooling kernels against plain PyTorch float32
on the same device (tolerance 1e-4 relative to the tensor scale, as BASELINE.json asks;
observed errors are ~1e-6)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from open3d_ml_b200 import _lib as L

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


@pytest.fixture(autouse=True)
def _kernel_routing(monkeypatch):
    """In this module the tensor-core kernel takes every aligned shape (the product routes K < 128 to
    the SIMT / row-per-thread kernels) and the row-per-thread kernel is off except in its own tests;
    restored afterwards so that the model tests see the product's routing."""
    monkeypatch.setattr(L, "TC_MIN_K", 8)
    monkeypatch.setattr(L, "USE_ROW_MLP", False)


def rnd(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).cuda()


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("n,cin,cout", [(1000, 8, 8), (4099, 3, 8), (777, 32, 19), (5000, 64, 64),
                                        (300, 768, 256), (2048, 128, 1024), (65, 75, 64), (1, 16, 13),
                                        (129, 40, 72), (70000, 256, 32),
                                        # short products on many row tiles: the two-CTAs-per-SM LITE kernels (gemm_tc.cu GtCfg)
                                        (30000, 64, 64), (20011, 96, 128), (40000, 128, 32)])
def test_linear_plain(n, cin, cout, tc):
    """tc=True: PackedWeight -> wgmma kernel (gemm_tc.cu) whenever cin % 8 == 0, SIMT otherwise."""
    x, w = rnd(n, cin, seed=1), rnd(cin, cout, seed=2) / cin ** 0.5
    s, t = rnd(cout, seed=3).abs() + 0.5, rnd(cout, seed=4)
    out = torch.full((n, cout), float("nan")).cuda()
    wk = L.pack_linear(w) if tc else w
    L.linear([L.make_src(x)], wk, out, s, t, act="leaky", slope=0.2)
    ref = F.leaky_relu((x.double() @ w.double()) * s + t, 0.2)
    assert rel_err(out, ref) < TOL
    L.linear([L.make_src(x)], wk, out, None, None, act=None)
    assert rel_err(out, x.double() @ w.double()) < TOL


@pytest.mark.parametrize("tc", [False, True])
def test_linear_concat_gather_residual_batched_index(tc):
    B, nup, nco = 3, 500, 120
    skip, coarse = rnd(B * nup, 32, seed=1), rnd(B * nco, 64, seed=2)
    idx = torch.randint(0, nco, (B, nup, 1), generator=torch.Generator().manual_seed(3)).cuda()
    w, t, res = rnd(96, 48, seed=4) / 10, rnd(48, seed=5), rnd(B * nup, 48, seed=6)
    out = torch.empty(B * nup, 48).cuda()
    L.linear([L.make_src(skip), L.make_src(coarse, index=idx.view(-1), out_rows_per_batch=nup,
                                           src_rows_per_batch=nco)], L.pack_linear(w) if tc else w, out, None, t,
             residual=res, act="relu")
    up = torch.gather(coarse.view(B, nco, 64), 1, idx.expand(-1, -1, 64)).reshape(B * nup, 64)
    ref = torch.relu(torch.cat([skip, up], 1) @ w + t + res)
    assert rel_err(out, ref) < TOL
    # global int32 index with shadow rows (== rows -> zeros), column 0 of a wider index matrix
    nq, ns = 700, 300
    x = rnd(ns, 24 if tc else 20, seed=7)
    nb = torch.randint(0, ns + 1, (nq, 5), generator=torch.Generator().manual_seed(8)).to(torch.int32).cuda()
    w2 = rnd(x.shape[1], 7, seed=9)
    out2 = torch.empty(nq, 7).cuda()
    L.linear([L.make_src(x, index=nb, index_ld=5)], L.pack_linear(w2) if tc else w2, out2, act=None)
    xz = torch.cat([x, torch.zeros(1, x.shape[1]).cuda()])
    assert rel_err(out2, xz[nb[:, 0].long()] @ w2) < TOL


@pytest.mark.parametrize("tc", [False, True])
def test_linear_nchw_output_and_strided_out(tc):
    B, H, W, C, Co = 2, 9, 7, 24, 10
    x, w, b = rnd(B * H * W, C, seed=1), rnd(C, Co, seed=2), rnd(Co, seed=3)
    out = torch.empty(B, Co, H, W).cuda()
    L.linear([L.make_src(x)], L.pack_linear(w) if tc else w, out, None, b, act=None, num_rows=B * H * W,
             out_channels=Co, out_nchw_plane=H * W)
    ref = (x @ w + b).view(B, H * W, Co).permute(0, 2, 1).reshape(B, Co, H, W)
    assert rel_err(out, ref) < TOL
    wide = torch.zeros(B * H * W, 40).cuda()                 # write 12 channels into columns 16..28
    w3 = rnd(C, 12, seed=4)
    L.linear([L.make_src(x)], L.pack_linear(w3) if tc else w3, wide[:, 16:28], act=None, num_rows=B * H * W,
             out_ld=40)
    assert rel_err(wide[:, 16:28], x @ w3) < TOL and float(wide[:, :16].abs().max()) == 0 and float(wide[:, 28:].abs().max()) == 0


# Against float64 on an H100 80GB HBM3 (400 W power limit), the largest rel_err of the convolutions and transposed
# convolutions below was 1.35e-6 (fp32 SIMT and 3xTF32 alike); the bound keeps about 5x of margin.
DENSE_TOL = 7e-6


def _conv3x3_case(B, H, W, C, Co, stride, tc, seed=1):
    """rel_err of conv3x3 (scale, shift, ReLU) against float64 torch; the output starts as NaN, so a pixel the kernel
    skips fails the comparison."""
    x = rnd(B, H, W, C, seed=seed)
    w = rnd(Co, C, 3, 3, seed=seed + 1) / (9 * C) ** 0.5
    s, t = rnd(Co, seed=seed + 2).abs() + 0.5, rnd(Co, seed=seed + 3)
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.full((B, OH, OW, Co), float("nan")).cuda()
    wt = w.permute(2, 3, 1, 0).reshape(9 * C, Co).contiguous()
    L.conv3x3(x, L.pack_linear(wt) if tc else wt, out, s, t, stride, act="relu")
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), None, stride, 1)
    ref = torch.relu(ref * s.double().view(1, -1, 1, 1) + t.double().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    assert ref.shape == out.shape
    return rel_err(out, ref)


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("B,H,W,C,Co,stride", [(1, 20, 16, 64, 64, 1), (2, 31, 27, 64, 128, 2),
                                                (1, 62, 54, 128, 128, 1), (1, 13, 13, 256, 256, 2)])
def test_conv3x3_nhwc(B, H, W, C, Co, stride, tc):
    assert _conv3x3_case(B, H, W, C, Co, stride, tc) < DENSE_TOL


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("H,W", [(h, w) for h in (1, 2, 3, 5) for w in (1, 2, 3, 5)])
def test_conv3x3_nhwc_small_images(H, W, stride, tc):
    """Images of 1 to 5 pixels a side, where every tap but the centre one reaches into the padding and a stride-2
    image may have no odd rows or columns (the tensor-core kernel loads each row / column parity through its own
    tensor map); output widths that are not a multiple of 32."""
    errs = {co: _conv3x3_case(3, H, W, 64, co, stride, tc, seed=co) for co in (8, 19, 64, 160)}
    assert max(errs.values()) < DENSE_TOL, errs


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("stride", [1, 2, 4])
@pytest.mark.parametrize("H,W,Co", [(6, 5, 128), (1, 5, 6), (4, 1, 10), (1, 1, 128), (3, 1, 6), (1, 2, 10)])
def test_deconv_nhwc_into_concat_buffer(H, W, Co, stride, tc):
    """Into a channel slice of a wider NaN-filled buffer whose other columns must keep their NaN.  Co % 4 != 0 takes
    the one-element-per-thread pixel shuffle of the tensor-core epilogue (gemm_tc.cu)."""
    assert _deconv_case(H, W, Co, stride, tc) < DENSE_TOL


def _deconv_case(H, W, Co, stride, tc):
    B, C, lo = 2, 64, 4
    x = rnd(B, H, W, C, seed=1)
    w = rnd(C, Co, stride, stride, seed=2) / C ** 0.5
    s, t = rnd(Co, seed=3).abs() + 0.5, rnd(Co, seed=4)
    neck = torch.full((B, H * stride, W * stride, Co + 12), float("nan")).cuda()
    wt = w.permute(0, 2, 3, 1).reshape(C, stride * stride * Co).contiguous()
    s_rep, t_rep = s.repeat(stride * stride), t.repeat(stride * stride)   # keep alive across the call
    L.deconv(x, L.pack_linear(wt) if tc else wt, neck[..., lo:lo + Co], s_rep, t_rep, stride, act="relu")
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2).double(), w.double(), None, stride)
    ref = torch.relu(ref * s.double().view(1, -1, 1, 1) + t.double().view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    assert bool(neck[..., :lo].isnan().all()) and bool(neck[..., lo + Co:].isnan().all())
    return rel_err(neck[..., lo:lo + Co], ref)


def test_gather_max_batched_and_shadow():
    B, N, ns, C, K = 2, 400, 100, 32, 16
    x = rnd(B * N, C, seed=1)
    idx = torch.randint(0, N, (B, ns, K), generator=torch.Generator().manual_seed(2)).cuda()
    out = torch.empty(B * ns, C).cuda()
    L.check(L.lib().o3dml_gather_max(L.ptr(x), B * N, C, C, L.ptr(idx), 1, B * ns, K, ns, N, 0, L.ptr(out), C, L.stream()))
    ref = torch.gather(x.view(B, N, C), 1, idx.view(B, ns * K, 1).expand(-1, -1, C)).view(B, ns, K, C).max(2)[0]
    assert torch.equal(out.view(B, ns, C), ref)
    x2 = -rnd(300, 8, seed=3).abs()                          # all negative: the shadow zero row must win
    nb = torch.randint(0, 301, (50, 6), generator=torch.Generator().manual_seed(4)).cuda()
    nb[0] = 300
    out2 = torch.empty(50, 8).cuda()
    L.check(L.lib().o3dml_gather_max(L.ptr(x2), 300, 8, 8, L.ptr(nb), 1, 50, 6, 0, 0, 1, L.ptr(out2), 8, L.stream()))
    ref2 = torch.cat([x2, torch.zeros(1, 8).cuda()])[nb].max(1)[0]
    assert torch.equal(out2, ref2) and float(out2[0].abs().max()) == 0


@pytest.mark.parametrize("cin,H", [(5, 27), (32, 35), (64, 40), (200, 7), (128, 33), (256, 20), (32, 3), (10, 9)])
def test_kpconv_gather_vs_torch(cin, H):
    from oracle import models_torch as MT
    nq, ns, K = 333, 500, 15
    g = torch.Generator().manual_seed(5)
    s_pts = torch.rand(ns, 3, generator=g).cuda()
    q_pts = s_pts[:nq] + 0.01 * torch.randn(nq, 3, generator=g).cuda()
    nb = torch.randint(0, ns + 1, (nq, H), generator=g).cuda()
    x, kp = rnd(ns, cin, seed=6), (torch.rand(K, 3, generator=g).cuda() - 0.5) * 0.3
    ext = 0.12
    a = torch.empty(nq, K * cin).cuda()
    L.check(L.lib().o3dml_kpconv_gather(L.ptr(q_pts), nq, L.ptr(s_pts), ns, L.ptr(nb), 1, H, L.ptr(x), cin,
                                        L.ptr(kp), K, ext, L.ptr(a), L.stream()))
    w = torch.eye(K * cin).view(K, cin, K * cin).cuda()      # identity weights expose the [K*Cin] tensor
    ref = MT.kp_conv(q_pts, s_pts, nb, x, kp, w, ext)
    assert rel_err(a, ref) < TOL


@pytest.mark.parametrize("mag", [1e-20, 1e-6, 1e-3, 1.0, 3e4, 1e20])
def test_linear_tc_is_magnitude_independent(mag):
    """The TF32 split keeps fp32's exponent (gemm_tc.cu): the relative error must not depend on the
    scale of the activations (an fp16 split would need a per-tile range normalisation for this)."""
    n, cin, cout = 3000, 256, 64
    x, w = rnd(n, cin, seed=1) * mag, rnd(cin, cout, seed=2) * 1e-3
    out = torch.empty(n, cout).cuda()
    L.linear([L.make_src(x)], L.pack_linear(w), out, act=None)
    assert rel_err(out, x.double() @ w.double()) < 3e-6


ROW_SHAPES = [(3, 0, 8), (8, 0, 8), (16, 0, 8), (16, 0, 16), (16, 8, 32), (32, 0, 32), (64, 0, 32), (64, 0, 64),
              (32, 32, 32), (32, 0, 64), (32, 0, 19)]


@pytest.mark.parametrize("c0,c1,co", ROW_SHAPES)
@pytest.mark.parametrize("n", [1, 257, 40000])
def test_linear_rows_small(c0, c1, co, n, monkeypatch):
    """rowmlp.cu (weights in the kernel parameter block, thread per row) vs float64 torch; the
    second source is gathered through a batch-relative index as in the RandLA-Net decoder."""
    monkeypatch.setattr(L, "USE_ROW_MLP", True)
    monkeypatch.setattr(L, "ROW_MLP_MIN_ROWS", 0)      # the product prefers the tensor-core kernel below 40 000 rows
    assert L.lib().o3dml_linear_rows_small_supported(c0, c1, co) == 1
    B = 2 if n > 1 else 1
    a = rnd(B * n, c0, seed=1)
    w = rnd(c0 + c1, co, seed=2) / (c0 + c1) ** 0.5
    s, t = rnd(co, seed=3).abs() + 0.5, rnd(co, seed=4)
    srcs, cols = [L.make_src(a)], [a.double()]
    if c1:
        nco = max(1, n // 3)
        coarse = rnd(B * nco, c1, seed=5)
        idx = torch.randint(0, nco, (B, n, 1), generator=torch.Generator().manual_seed(6)).cuda()
        srcs.append(L.make_src(coarse, index=idx.view(-1), out_rows_per_batch=n, src_rows_per_batch=nco))
        cols.append(torch.gather(coarse.view(B, nco, c1), 1, idx.expand(-1, -1, c1)).reshape(B * n, c1).double())
    pw = L.pack_linear(w)
    n0 = L.lib().o3dml_launch_count()
    out = torch.full((B * n, co), float("nan")).cuda()
    L.linear(srcs, pw, out, s, t, act="leaky", slope=0.2)
    assert L.lib().o3dml_launch_count() == n0 + 1
    ref = F.leaky_relu((torch.cat(cols, 1) @ w.double()) * s + t, 0.2)
    assert rel_err(out, ref) < TOL
    out2 = torch.full((B * n, co), float("nan")).cuda()
    L.linear(srcs, pw, out2, None, t, act=None)
    assert rel_err(out2, torch.cat(cols, 1) @ w.double() + t) < TOL


def test_linear_rows_small_rejects_unsupported_shape_and_device_weights():
    x = rnd(100, 24, seed=1)
    arr = (L.Src * 1)(L.make_src(x))
    out = torch.empty(100, 8).cuda()
    w = torch.zeros(24, 8)
    assert L.lib().o3dml_linear_rows_small_supported(24, 0, 8) == 0
    rc = L.lib().o3dml_linear_rows_small(100, arr, 1, w.data_ptr(), None, None, 0, 0.0, L.ptr(out), 8, 8, L.stream())
    assert rc != 0
    x8 = rnd(100, 8, seed=2)
    arr = (L.Src * 1)(L.make_src(x8))
    rc = L.lib().o3dml_linear_rows_small(100, arr, 1, torch.zeros(8, 8).cuda().data_ptr(), None, None, 0, 0.0,
                                         L.ptr(out), 8, 8, L.stream())
    assert rc != 0
    with pytest.raises(RuntimeError):
        L.check(rc)


def test_linear_tc_three_sources_mixed_tma_and_gather():
    """identity (TMA) | gathered with shadow rows (cp.async) | identity with a ragged 24-channel tail (TMA
    zero fill beyond the tensor) in one GEMM; 1000 rows = 7 full tiles + a 104-row tail."""
    n, ns = 1000, 300
    a, b, c = rnd(n, 64, seed=1), rnd(ns, 32, seed=2), rnd(n, 24, seed=3)
    nb = torch.randint(0, ns + 1, (n, 3), generator=torch.Generator().manual_seed(4)).cuda()
    w = rnd(120, 40, seed=5) / 11
    out = torch.full((n, 40), float("nan")).cuda()
    L.linear([L.make_src(a), L.make_src(b, index=nb, index_ld=3), L.make_src(c)], L.pack_linear(w), out, act=None)
    bz = torch.cat([b, torch.zeros(1, 32).cuda()])[nb[:, 0]]
    ref = torch.cat([a, bz, c], 1).double() @ w.double()
    assert rel_err(out, ref) < 3e-6


def test_linear_tc_strided_source_view():
    """A column slice of a wider buffer as the operand (ld > channels): the tensor map carries the stride."""
    wide = rnd(5000, 96, seed=1)
    w = rnd(64, 128, seed=2) / 8
    out = torch.empty(5000, 128).cuda()
    L.linear([L.make_src(wide[:, 32:], channels=64, ld=96)], L.pack_linear(w), out, act=None)
    assert rel_err(out, wide[:, 32:].double() @ w.double()) < 3e-6


def _gathered(data, n, index=None, index_ld=1, out_rows_per_batch=0, src_rows_per_batch=0):
    """float64 rows that output rows 0..n-1 read from a source (include/o3dml_b200.h o3dml_src_t; index_ld <= 0 reads
    as 1): row n itself, or the row its index names, zeros where the id is negative, past src_rows_per_batch
    (batch-relative) or where the resolved row is not in [0, rows)."""
    if index is None:
        return data[:n].double()
    r = index.reshape(-1)[::max(index_ld, 1)][:n].long()
    ok = r >= 0
    if out_rows_per_batch > 0:
        ok &= r < src_rows_per_batch
        r = r + (torch.arange(n, device=r.device) // out_rows_per_batch) * src_rows_per_batch
    ok &= r < data.shape[0]
    out = torch.zeros(n, data.shape[1], dtype=torch.float64, device=data.device)
    out[ok] = data[r[ok]].double()
    return out


def _dense_case(name, n):
    """Two 32-channel sources of the (32 + 32) -> 32 layer: a list of make_src keyword sets (data first)."""
    g = torch.Generator().manual_seed(11)
    a, b = rnd(n, 32, seed=12), rnd(n, 32, seed=13)
    pool = rnd(300, 32, seed=14)
    if name == "identity":
        return [dict(data=a), dict(data=b)]
    if name == "global_int32_column0":               # column 0 of an [n, 3] id matrix
        nb = torch.randint(0, 300, (n, 3), generator=g).to(torch.int32).cuda()
        return [dict(data=a), dict(data=pool, index=nb, index_ld=3)]
    if name == "shadow_ids":                        # ids -1 and == rows read zeros, in both sources
        i0 = torch.randint(-1, 301, (n,), generator=g).cuda()
        i1 = torch.randint(-1, 301, (n, 2), generator=g).to(torch.int32).cuda()
        i0[:2], i1[:2, 0] = torch.tensor([-1, 300]).cuda(), torch.tensor([300, -1], dtype=torch.int32).cuda()
        return [dict(data=pool, index=i0), dict(data=pool, index=i1, index_ld=2)]
    if name == "batch_relative_int64":               # ids == src_rows_per_batch and past it read zeros
        B, nco = 2, 150
        idx = torch.randint(0, nco + 2, (n,), generator=g).cuda()
        idx[:2] = torch.tensor([nco, nco + 1]).cuda()
        return [dict(data=a), dict(data=pool, index=idx, out_rows_per_batch=n // B, src_rows_per_batch=nco)]
    if name == "index_ld0":                         # index_ld = 0 reads as 1
        idx = torch.randint(0, 300, (n,), generator=g).to(torch.int32).cuda()
        return [dict(data=pool, index=idx, index_ld=0), dict(data=b)]
    raise KeyError(name)


ROUTES = {   # _lib.linear's choice for a PackedWeight, forced through its routing constants
    "simt": ("o3dml_linear", dict(TC_MIN_K=10 ** 9, USE_ROW_MLP=False)),
    "tc": ("o3dml_linear_tc", dict(TC_MIN_K=8, USE_ROW_MLP=False)),
    "rows_small": ("o3dml_linear_rows_small", dict(USE_ROW_MLP=True, ROW_MLP_MIN_ROWS=0)),
}


@pytest.mark.parametrize("case", ["identity", "global_int32_column0", "shadow_ids", "batch_relative_int64",
                                  "index_ld0"])
@pytest.mark.parametrize("route", list(ROUTES))
def test_linear_routes_read_sources_alike(route, case, monkeypatch):
    """The same gathered sources through each of linear's three kernels (gemm.cu, gemm_tc.cu, rowmlp.cu) vs float64."""
    n = 1000
    entry, consts = ROUTES[route]
    for k, v in consts.items():
        monkeypatch.setattr(L, k, v)
    h, called = L.lib(), []
    for name in ("o3dml_linear", "o3dml_linear_tc", "o3dml_linear_rows_small"):
        fn = getattr(h, name)
        monkeypatch.setattr(h, name, lambda *a, _fn=fn, _name=name: called.append(_name) or _fn(*a))
    kws = _dense_case(case, n)
    srcs = [L.make_src(**kw) for kw in kws]
    x = torch.cat([_gathered(kw["data"], n, kw.get("index"), kw.get("index_ld", 1), kw.get("out_rows_per_batch", 0),
                             kw.get("src_rows_per_batch", 0)) for kw in kws], 1)
    w = rnd(64, 32, seed=15) / 8
    s, t = rnd(32, seed=16).abs() + 0.5, rnd(32, seed=17)
    out = torch.full((n, 32), float("nan")).cuda()
    n0 = L.lib().o3dml_launch_count()
    L.linear(srcs, L.pack_linear(w), out, s, t, act="leaky", slope=0.2)
    assert L.lib().o3dml_launch_count() == n0 + 1 and called == [entry]
    ref = F.leaky_relu((x @ w.double()) * s + t, 0.2)
    assert rel_err(out, ref) < TOL


def test_linear_rows_small_rejects_malformed_sources():
    """rowmlp.cu takes the source checks of o3dml_linear: ld < channels and null data are errors, not launches."""
    x = rnd(101, 32, seed=1)
    out = torch.empty(100, 32).cuda()
    w = torch.zeros(32, 32)
    narrow, null = L.make_src(x, channels=32, ld=16, rows=100), L.make_src(x, rows=100)
    null.data = None
    for src in (narrow, null):
        n0 = L.lib().o3dml_launch_count()
        rc = L.lib().o3dml_linear_rows_small(100, (L.Src * 1)(src), 1, w.data_ptr(), None, None, 0, 0.0, L.ptr(out),
                                             32, 32, L.stream())
        assert rc != 0 and L.lib().o3dml_launch_count() == n0
        with pytest.raises(RuntimeError):
            L.check(rc)
