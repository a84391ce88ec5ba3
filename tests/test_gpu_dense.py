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


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("B,H,W,C,Co,stride", [(1, 20, 16, 64, 64, 1), (2, 31, 27, 64, 128, 2),
                                                (1, 62, 54, 128, 128, 1), (1, 13, 13, 256, 256, 2)])
def test_conv3x3_nhwc(B, H, W, C, Co, stride, tc):
    x = rnd(B, H, W, C, seed=1)
    w = rnd(Co, C, 3, 3, seed=2) / (9 * C) ** 0.5
    s, t = rnd(Co, seed=3).abs() + 0.5, rnd(Co, seed=4)
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.empty(B, OH, OW, Co).cuda()
    wt = w.permute(2, 3, 1, 0).reshape(9 * C, Co).contiguous()
    if tc:
        pw = L.pack_linear(wt)
        L.check(L.lib().o3dml_conv3x3_nhwc_tc(L.ptr(x), B, H, W, C, stride, L.ptr(pw.img), pw.k_pad, pw.n_pad,
                                              L.ptr(s), L.ptr(t), 1, 0.0, L.ptr(out), Co, L.stream()))
    else:
        L.check(L.lib().o3dml_conv3x3_nhwc(L.ptr(x), B, H, W, C, stride, L.ptr(wt), L.ptr(s), L.ptr(t), 1, 0.0,
                                           L.ptr(out), Co, L.stream()))
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, None, stride, 1)
    ref = torch.relu(ref * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    assert ref.shape == out.shape and rel_err(out, ref) < TOL


@pytest.mark.parametrize("tc", [False, True])
@pytest.mark.parametrize("stride", [1, 2, 4])
def test_deconv_nhwc_into_concat_buffer(stride, tc):
    B, H, W, C, Co = 2, 6, 5, 64, 128
    x = rnd(B, H, W, C, seed=1)
    w = rnd(C, Co, stride, stride, seed=2) / C ** 0.5
    s, t = rnd(Co, seed=3).abs() + 0.5, rnd(Co, seed=4)
    neck = torch.zeros(B, H * stride, W * stride, 384).cuda()
    wt = w.permute(0, 2, 3, 1).reshape(C, stride * stride * Co).contiguous()
    s_rep, t_rep = s.repeat(stride * stride), t.repeat(stride * stride)   # keep alive across the call
    if tc:
        pw = L.pack_linear(wt)
        L.check(L.lib().o3dml_deconv_nhwc_tc(L.ptr(x), B, H, W, C, stride, L.ptr(pw.img), pw.k_pad, pw.n_pad,
                                             L.ptr(s_rep), L.ptr(t_rep), 1, 0.0, neck.data_ptr() + 4 * 128, 384,
                                             Co, L.stream()))
    else:
        L.check(L.lib().o3dml_deconv_nhwc(L.ptr(x), B, H, W, C, stride, L.ptr(wt), L.ptr(s_rep), L.ptr(t_rep), 1,
                                          0.0, neck.data_ptr() + 4 * 128, 384, Co, L.stream()))
    ref = F.conv_transpose2d(x.permute(0, 3, 1, 2), w, None, stride)
    ref = torch.relu(ref * s.view(1, -1, 1, 1) + t.view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    assert rel_err(neck[..., 128:256], ref) < TOL
    assert float(neck[..., :128].abs().max()) == 0 and float(neck[..., 256:].abs().max()) == 0


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
