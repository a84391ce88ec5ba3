import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    # GPU tests never run (not even "skip") unless a device is visible
    try:
        import torch
        has = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        has = False
    if has:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


def rel_err(a, b):
    """max |a-b| / max |b| -- the 1e-4 'rel' of BASELINE.json's north_star."""
    import torch
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def elem_err(a, b, q=0.999, floor=1e-3):
    """Element-wise companion of rel_err: the q-quantile of |a-b| / (|b| + floor * max|b|).  rel_err is relative to the
    tensor scale, so a regression confined to small-magnitude entries (logits near zero) cannot move it; here every
    element is judged against its own magnitude down to `floor` of the scale."""
    import torch
    a, b = torch.as_tensor(a).double().cpu().reshape(-1), torch.as_tensor(b).double().cpu().reshape(-1)
    scale = b.abs().max().clamp_min(1e-30)
    r = (a - b).abs() / (b.abs() + floor * scale)
    if r.numel() > 4_000_000:                      # torch.quantile is limited to 16 M elements; sample evenly
        r = r[:: r.numel() // 4_000_000 + 1]
    return float(torch.quantile(r, q))
