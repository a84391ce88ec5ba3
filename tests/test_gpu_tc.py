"""wgmma bring-up: the descriptor encodings / operand layout of tc.cuh against torch."""
import pytest
import torch

from open3d_ml_b200 import _lib as L

pytestmark = pytest.mark.gpu


def run(n, k, terms, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(128, k, generator=g) * scale).cuda()
    b = (torch.randn(n, k, generator=g) / k ** 0.5).cuda()
    d = torch.full((128, n), float("nan")).cuda()
    L.check(L.lib().o3dml_tc_gemm_test(L.ptr(a), L.ptr(b), L.ptr(d), n, k, terms, L.stream()))
    torch.cuda.synchronize()
    ref = a.double() @ b.double().t()
    return float((d.double() - ref).abs().max() / ref.abs().max()), d, ref


@pytest.mark.parametrize("n,k", [(16, 16), (64, 64), (128, 128), (256, 128), (256, 64), (32, 256), (16, 320)])
def test_tc_gemm_3xfp16_matches_fp64(n, k):
    err, _, _ = run(n, k, 3)
    assert err < 2e-6, err


def test_tc_gemm_single_term_is_fp16_accurate_only():
    err1, _, _ = run(128, 128, 1)
    err3, _, _ = run(128, 128, 3)
    assert 1e-5 < err1 < 3e-3 and err3 < 2e-6


def test_tc_gemm_large_and_tiny_magnitudes():
    assert run(64, 64, 3, seed=1, scale=1e3)[0] < 2e-6
    assert run(64, 64, 3, seed=2, scale=1e-3)[0] < 1e-4      # lo parts are fp16-subnormal here
