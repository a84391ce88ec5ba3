"""Each entry that takes a workspace runs in exactly the bytes its *_workspace_bytes returns, on shapes that reach the
scratch paths: scans above one 4 096-element tile (the look-back path, which uses its temp), radix sorts over several
2 048-key blocks, batches with an empty item, NMS over more than 64 boxes, box decoding with and without top-k
selection.  The exact workspace sits at the front of a larger buffer whose tail holds a byte pattern: the outputs must
be bit-equal to those of a run with twice the workspace, and the tail must be untouched.  One byte less is refused
(status 2) before anything is enqueued."""
import pytest
import torch

from open3d_ml_b200 import _lib as L
from abi_cases import knn_case, nms_case, pp_detect_case, radius_case, sparse_conv_case, voxelize_case

pytestmark = pytest.mark.gpu

TAIL, PATTERN = 4096, 0xA5

CASES = {
    "voxelize": lambda: voxelize_case(splits=(0, 20000, 20000, 40000), voxel=0.1, max_voxels=30000),
    "knn": lambda: knn_case(p_splits=(0, 3000, 3000, 6000), q_splits=(0, 2500, 5000, 5000)),
    "radius": lambda: radius_case(p_splits=(0, 3000, 3000, 6000), q_splits=(0, 2500, 5000, 5000), radius=0.3),
    "sparse_conv_neighbors": lambda: sparse_conv_case(5000),
    "sparse_conv_neighbors_no_inputs": lambda: sparse_conv_case(0),
    "nms": lambda: nms_case(3000),
    "pp_detect": lambda: pp_detect_case(False),
    "pp_detect_select": lambda: pp_detect_case(True),
}


def calls(case):
    """The entries a case runs, in order: o3dml_radius_fill follows o3dml_radius_count on the same workspace."""
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


@pytest.mark.parametrize("name", list(CASES))
def test_exact_workspace_suffices_and_one_byte_less_is_refused(name):
    case = CASES[name]()
    wsb = case.wsb
    big = torch.empty(2 * wsb, dtype=torch.uint8, device="cuda")
    want = run(case, L.ptr(big), 2 * wsb)

    buf = torch.full((wsb + TAIL,), PATTERN, dtype=torch.uint8, device="cuda")
    got = run(case, L.ptr(buf), wsb)
    for a, b in zip(got, want):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name
    assert bool((buf[wsb:] == PATTERN).all()), "%s wrote past its %d-byte workspace" % (name, wsb)

    n0 = L.lib().o3dml_launch_count()
    for call in calls(case):
        assert call(L.ptr(buf), wsb - 1) == 2, L.lib().o3dml_last_error().decode()
        assert ("(%d needed)" % wsb) in L.lib().o3dml_last_error().decode()
    assert L.lib().o3dml_launch_count() == n0
