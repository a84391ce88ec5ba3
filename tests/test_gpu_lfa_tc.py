"""The wgmma LFA kernel (lfa_tc.cu) against the FP32 SIMT kernel (lfa.cu) on identical
inputs, and end-to-end through the model (the golden / port parity tests in
test_gpu_models.py run with the tensor-core path enabled by default)."""
import numpy as np
import pytest
import torch

from open3d_ml_b200 import _lib as L
from conftest import rel_err

pytestmark = pytest.mark.gpu


def make(d, B, N, seed, gain=1.0):
    g = torch.Generator().manual_seed(seed)
    h = d // 2
    coords = (torch.rand(B * N, 3, generator=g) * 10).cuda()
    nidx = torch.randint(0, N, (B, N, 16), generator=g).cuda()
    feat = torch.randn(B * N, h, generator=g).cuda()
    w10 = (torch.randn(10, h, generator=g) * 0.3).cuda()
    s10, t10 = (torch.rand(h, generator=g) + 0.5).cuda(), (torch.randn(h, generator=g) * 0.1).cuda()
    wl2 = (torch.randn(h, h, generator=g) / h ** 0.5)          # [out, in]
    s2, t2 = (torch.rand(h, generator=g) + 0.5).cuda(), (torch.randn(h, generator=g) * 0.1).cuda()
    ws = (torch.randn(d, d, generator=g) / d ** 0.5) * gain    # [out, in]; gain spreads the scores
    bs = torch.randn(d, generator=g).cuda()
    return coords, nidx, feat, w10, s10, t10, wl2, s2, t2, ws, bs


@pytest.mark.parametrize("d", [16, 32, 64, 128, 256])
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("B,N,gain", [(1, 8, 1.0), (2, 1000, 1.0), (3, 2817, 1.0), (2, 500, 40.0)])
def test_lfa_tc_matches_simt(d, stage, B, N, gain):
    """gain = 40 makes the scores of neighbouring points differ by hundreds: the softmax max must be
    taken per point (a wrong group maximum only shows up once exp() underflows)."""
    coords, nidx, feat, w10, s10, t10, wl2, s2, t2, ws, bs = make(d, B, N, 7 * d + stage, gain)
    ref = torch.full((B * N, d), float("nan")).cuda()
    out = torch.full((B * N, d), float("nan")).cuda()
    wl2t, wst = wl2.t().contiguous().cuda(), ws.t().contiguous().cuda()
    L.check(L.lib().o3dml_randla_lfa_pool(stage, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                          L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(wl2t), L.ptr(s2), L.ptr(t2),
                                          L.ptr(wst), L.ptr(bs), L.ptr(ref), L.stream()))
    img_l2 = L.pack_operand_image(wl2) if d >= 32 else None
    img_s = L.pack_operand_image(ws)
    L.check(L.lib().o3dml_randla_lfa_pool_tc(stage, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                             L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(img_l2), L.ptr(wl2t),
                                             L.ptr(s2), L.ptr(t2), L.ptr(img_s), L.ptr(out), L.stream()))
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert rel_err(out, ref) < (2e-5 if gain == 1.0 else 2e-3), rel_err(out, ref)


def lfa_reference(stage, d, coords, nidx, feat, w10, s10, t10, wl2, s2, t2, ws, bs, B, N):
    """float64 torch restatement of LocalSpatialEncoding + AttentivePooling score/softmax/sum
    (randlanet.py:521-639 as used at :667-692) on the same folded-BN parameters."""
    f64 = lambda t: t.detach().cpu().double()
    c = f64(coords).view(B, N, 3)
    idx = nidx.cpu()
    nbc = torch.stack([c[b][idx[b]] for b in range(B)])            # [B, N, 16, 3]
    q = c.unsqueeze(2).expand_as(nbc)
    rel = q - nbc
    enc = torch.cat([rel.pow(2).sum(-1, keepdim=True).sqrt(), rel, q, nbc], -1)
    lrelu = torch.nn.functional.leaky_relu
    r = lrelu(enc @ f64(w10) * f64(s10) + f64(t10), 0.2)
    if stage == 2:
        r = lrelu(r @ f64(wl2).t() * f64(s2) + f64(t2), 0.2)
    f = f64(feat).view(B, N, d // 2)
    fn = torch.stack([f[b][idx[b]] for b in range(B)])
    X = torch.cat([fn, r], -1)
    p = torch.softmax(X @ f64(ws).t() + f64(bs), dim=2)
    return (p * X).sum(2).reshape(B * N, d)


@pytest.mark.parametrize("d", [16, 32, 64, 128, 256])
@pytest.mark.parametrize("stage", [1, 2])
def test_lfa_kernels_vs_float64_reference(d, stage):
    """Every LFA implementation (FP32 SIMT, parameter-block d = 16, wgmma) against float64 torch;
    tolerance 1e-4 relative to the tensor scale (north_star), measured values are ~1e-6."""
    B, N = 2, 700
    args = make(d, B, N, 100 + d + stage)
    coords, nidx, feat, w10, s10, t10, wl2, s2, t2, ws, bs = args
    want = lfa_reference(stage, d, *args, B, N)
    wl2t, wst = wl2.t().contiguous().cuda(), ws.t().contiguous().cuda()
    outs = {}
    o = torch.full((B * N, d), float("nan")).cuda()
    L.check(L.lib().o3dml_randla_lfa_pool(stage, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                          L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(wl2t), L.ptr(s2), L.ptr(t2),
                                          L.ptr(wst), L.ptr(bs), L.ptr(o), L.stream()))
    outs["simt"] = o
    o = torch.full((B * N, d), float("nan")).cuda()
    img_l2 = L.pack_operand_image(wl2) if d >= 32 else None
    img_s = L.pack_operand_image(ws)
    L.check(L.lib().o3dml_randla_lfa_pool_tc(stage, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                             L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(img_l2), L.ptr(wl2t),
                                             L.ptr(s2), L.ptr(t2), L.ptr(img_s), L.ptr(o), L.stream()))
    outs["tc"] = o
    if d == 16:
        hw = torch.cat([w10.cpu().reshape(-1), s10.cpu(), t10.cpu(), wl2t.cpu().reshape(-1), s2.cpu(), t2.cpu(),
                        wst.cpu().reshape(-1), bs.cpu()]).contiguous()
        assert hw.numel() == 448
        o = torch.full((B * N, d), float("nan")).cuda()
        L.check(L.lib().o3dml_randla_lfa16_pool(stage, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                                hw.data_ptr(), L.ptr(o), L.stream()))
        outs["param_block"] = o
    torch.cuda.synchronize()
    for name, got in outs.items():
        assert rel_err(got.cpu().double(), want) < 1e-4, (name, rel_err(got.cpu().double(), want))


def test_lfa16_rejects_device_weights():
    coords, nidx, feat, *_ = make(16, 1, 64, 5)
    o = torch.empty(64, 16).cuda()
    rc = L.lib().o3dml_randla_lfa16_pool(1, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), 1, 64,
                                         torch.zeros(448).cuda().data_ptr(), L.ptr(o), L.stream())
    assert rc != 0
    with pytest.raises(RuntimeError):
        L.check(rc)


@pytest.mark.parametrize("stage", [1, 2])
def test_lfa_simt_d512_vs_float64_reference(stage):
    """d_out = 512 (fifth encoder of the s3dis / semantic3d / toronto3d / parislille3d configs,
    randlanet_s3dis.yml: dim_output [16, 64, 128, 256, 512]) runs on the FP32 SIMT kernel."""
    d, B, N = 512, 2, 150
    args = make(d, B, N, 900 + stage)
    coords, nidx, feat, w10, s10, t10, wl2, s2, t2, ws, bs = args
    want = lfa_reference(stage, d, *args, B, N)
    wl2t, wst = wl2.t().contiguous().cuda(), ws.t().contiguous().cuda()
    o = torch.full((B * N, d), float("nan")).cuda()
    L.check(L.lib().o3dml_randla_lfa_pool(stage, d, L.ptr(coords), L.ptr(nidx), 1, 16, L.ptr(feat), B, N,
                                          L.ptr(w10), L.ptr(s10), L.ptr(t10), L.ptr(wl2t), L.ptr(s2), L.ptr(t2),
                                          L.ptr(wst), L.ptr(bs), L.ptr(o), L.stream()))
    torch.cuda.synchronize()
    assert rel_err(o.cpu().double(), want) < 1e-4
