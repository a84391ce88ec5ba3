"""Each entry that takes a workspace runs in exactly the bytes its *_workspace_bytes returns, on shapes that reach the
scratch paths: scans above one 4 096-element tile (the look-back path, which uses its temp), radix sorts over several
2 048-key blocks, batches with an empty item, NMS over more than 64 boxes, box decoding with and without top-k
selection.  The exact workspace sits at the front of a larger buffer whose tail holds a byte pattern: the outputs must
be bit-equal to those of a run with twice the workspace, and the tail must be untouched.  Where a case has an oracle,
the outputs must equal it too; a k-NN output whose rows are packed at its front is compared over their length.  One
byte less is refused (status 2) before anything is enqueued.  The cases are abi_cases.WORKSPACE_CASES."""
import numpy as np
import pytest
import torch

from open3d_ml_b200 import _lib as L
from abi_cases import WORKSPACE_CASES

pytestmark = pytest.mark.gpu

TAIL, PATTERN = 4096, 0xA5


def calls(case):
    """The entries a case runs, in order: a fill follows its count on the same workspace."""
    return [case.run, case.fill] if hasattr(case, "fill") else [case.run]


def run(case, ws, nbytes):
    """Copies of everything the case's calls write, with the workspace at device address ws."""
    for t in case.outputs:
        t.zero_()
    L.check(case.run(ws, nbytes))
    out = [t.clone() for t in case.outputs]
    if hasattr(case, "fill"):
        case.prepare_fill()
        L.check(case.fill(ws, nbytes))
        out += [t.clone() for t in case.fill_outputs]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", list(WORKSPACE_CASES))
def test_exact_workspace_suffices_and_one_byte_less_is_refused(name):
    sizing, build = WORKSPACE_CASES[name]
    case = build()
    assert case.sizing == sizing, name
    wsb = case.wsb
    big = torch.empty(2 * wsb, dtype=torch.uint8, device="cuda")
    want = run(case, L.ptr(big), 2 * wsb)

    buf = torch.full((wsb + TAIL,), PATTERN, dtype=torch.uint8, device="cuda")
    got = run(case, L.ptr(buf), wsb)
    for a, b in zip(got, want):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name
    assert bool((buf[wsb:] == PATTERN).all()), "%s wrote past its %d-byte workspace" % (name, wsb)
    if case.reference:
        ref = case.reference()
        assert len(ref) == len(got), name
        for i, (a, r) in enumerate(zip(got, ref)):
            assert np.array_equal(a.cpu().numpy()[:len(r)], r), "%s: output %d differs from the oracle" % (name, i)

    n0 = L.lib().o3dml_launch_count()
    for call in calls(case):
        assert call(L.ptr(buf), wsb - 1) == 2, L.lib().o3dml_last_error().decode()
        assert ("(%d needed)" % wsb) in L.lib().o3dml_last_error().decode()
    assert L.lib().o3dml_launch_count() == n0
