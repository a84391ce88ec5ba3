"""The 3xFP16 split arithmetic of the tensor-core kernels (csrc/tc.cuh, gemm_tc.cu, lfa_tc.cu), emulated in
numpy on the CPU: x = hi + lo with hi = fp16(x), lo = fp16(x - hi); A.B ~ A_hi.B_hi + A_hi.B_lo + A_lo.B_hi
accumulated in fp32.  These tests pin (a) the host-side operand image layout, (b) the error level the
kernels are designed for (~1e-6 of the result scale, 100x inside the 1e-4 parity bar), and (c) why both
operands are range-normalised by exact powers of two before the split."""
import math

import numpy as np
import torch

from open3d_ml_b200 import _lib as L
from conftest import rel_err


def split(x):
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32), lo.astype(np.float32)


def gemm_3xfp16(a, b):
    """[M,K] x [K,N] with the three-product split, fp32 accumulation (numpy matmul on float32)."""
    ah, al = split(a)
    bh, bl = split(b)
    return (ah @ bh) + (ah @ bl) + (al @ bh)


def pow2_scale(x, target=13):
    m = float(np.abs(x).max())
    e = target - math.floor(math.log2(m)) if 0.0 < m < 3e38 else 0
    return e, x * np.float32(2.0 ** e)


def test_operand_image_layout_and_precision():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(24, 40, generator=g) * 3.0                       # [N, K]
    img = L.pack_operand_image_host(w).view(torch.float16)
    n, k = w.shape
    hi = img[: n * k].view(k // 8, n, 8).permute(1, 0, 2).reshape(n, k).float()
    lo = img[n * k:].view(k // 8, n, 8).permute(1, 0, 2).reshape(n, k).float()
    assert torch.equal(hi, w.to(torch.float16).float())              # chunk-major [K/8][N][8]
    # hi + lo carries 22 mantissa bits of w
    assert float(((hi + lo) - w).abs().max() / w.abs().max()) < 2.0 ** -21
    # chunk c of row r sits at uint4 index c * N + r (what the wgmma descriptor's LBO = N * 16 B assumes)
    u = img[: n * k].view(k // 8, n, 8)
    assert torch.equal(u[3, 5], w[5, 24:32].to(torch.float16))


def test_split_product_error_is_1e6_of_scale():
    rng = np.random.default_rng(1)
    a = rng.standard_normal((256, 2304)).astype(np.float32)
    b = (rng.standard_normal((2304, 128)) / 48).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    got = gemm_3xfp16(a, b)
    assert rel_err(got, ref) < 3e-6
    # plain fp16 (one product) is ~1000x worse: the reason for the split
    one = split(a)[0] @ split(b)[0]
    assert rel_err(one, ref) > 1e-4


def test_small_magnitudes_need_range_normalisation():
    """lo parts of |x| < 2^-3 are subnormal halves (and 0 below 2^-24): without the power-of-two
    normalisation of gemm_tc.cu / _lib.PackedWeight the error grows to the 1e-4 level."""
    rng = np.random.default_rng(2)
    a = (rng.standard_normal((128, 512)) * 1e-4).astype(np.float32)
    b = (rng.standard_normal((512, 64)) * 1e-3).astype(np.float32)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    raw = gemm_3xfp16(a, b)
    ea, an = pow2_scale(a)
    eb, bn = pow2_scale(b)
    assert 2.0 ** 13 <= float(np.abs(an).max()) < 2.0 ** 14
    norm = gemm_3xfp16(an, bn) * np.float32(2.0 ** (-ea - eb))      # exact un-scaling
    assert rel_err(norm, ref) < 3e-6
    assert rel_err(raw, ref) > 10 * rel_err(norm, ref)


def test_packed_weight_exponent_matches_the_kernel_contract():
    w = torch.randn(96, 40, generator=torch.Generator().manual_seed(3)) * 0.02    # [K, Cout]
    wmax = float(w.abs().max())
    e = int(13 - math.floor(math.log2(wmax)))
    assert 2.0 ** 13 <= wmax * 2.0 ** e < 2.0 ** 14
    # the image PackedWeight builds is pack_operand_image_host of the padded, scaled [Cout_pad, K_pad] matrix
    k_pad, n_pad = 96, 64
    wp = torch.zeros(n_pad, k_pad)
    wp[:40, :96] = w.t() * 2.0 ** e
    img = L.pack_operand_image_host(wp).view(torch.float16)
    hi = img[: n_pad * k_pad].view(k_pad // 8, n_pad, 8).permute(1, 0, 2).reshape(n_pad, k_pad).float()
    lo = img[n_pad * k_pad:].view(k_pad // 8, n_pad, 8).permute(1, 0, 2).reshape(n_pad, k_pad).float()
    assert float(((hi + lo)[:40, :96] * 2.0 ** -e - w.t()).abs().max() / wmax) < 2.0 ** -21
    assert float((hi + lo)[40:].abs().max()) == 0.0                                # zero padding


# ---- the 3xTF32 split of gemm_tc.cu -------------------------------------------------------------------
def _tf32_trunc(x):
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def test_tf32_split_three_products_reach_2e_minus_6():
    """Emulates gemm_tc.cu: A: hi = x & 0xFFFFE000, lo = x - hi (the tensor core truncates lo to TF32);
    W: host-side round-to-nearest split (_lib.pack_tf32_image_host); products accumulated in float64
    here (the kernel's fp32 accumulation adds its own ~1e-7).  No range normalisation is needed: the
    error does not depend on the magnitude of the operands."""
    import torch
    from open3d_ml_b200 import _lib as L
    rng = np.random.default_rng(0)
    for mag in (1e-20, 1e-6, 1.0, 3e4, 1e20):
        a = (rng.standard_normal((64, 256)) * mag).astype(np.float32)
        w = (rng.standard_normal((256, 32)) / 16).astype(np.float32)
        img = L.pack_tf32_image_host(torch.from_numpy(np.ascontiguousarray(w.T))).numpy()
        wh, wl = img[:32].T.astype(np.float64), img[32:].T.astype(np.float64)
        assert np.array_equal(_tf32_trunc(img), img)                 # both images are TF32-exact
        ah = _tf32_trunc(a)
        al = _tf32_trunc(a - ah)                                     # exact subtraction, then HW truncation
        ref = a.astype(np.float64) @ w.astype(np.float64)
        got = ah.astype(np.float64) @ wh + ah.astype(np.float64) @ wl + al.astype(np.float64) @ wh
        one = ah.astype(np.float64) @ wh
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() / scale < 2e-6
        assert np.abs(one - ref).max() / scale > 2e-5                # a single TF32 product is not enough


def test_tf32_round_is_nearest_even():
    import torch
    from open3d_ml_b200 import _lib as L
    x = torch.tensor([1.0, 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, 1.0 + 3 * 2.0 ** -11, -1.0 - 2.0 ** -10,
                      0.0, 65504.0, 3.0e38], dtype=torch.float32)
    r = L.tf32_round(x)
    exp = torch.tensor([1.0, 1.0, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -9, -1.0 - 2.0 ** -10, 0.0, 65504.0, 3.0e38])
    exp[-1] = r[-1]
    assert torch.equal(r[:-1], exp[:-1]) and abs(float(r[-1]) / 3.0e38 - 1) < 1e-3
