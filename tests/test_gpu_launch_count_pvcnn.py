"""o3dml_launch_count() against the kernels the GPU actually ran, for the PVCNN entries (abi_cases_pvcnn.LAUNCH_CASES):
what tests/test_gpu_launch_count.py checks for the entries of o3dml_b200.h.  The module is named to run right after
that one, so that all profiling sessions of a test process follow one another."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", ["pv_voxel_cells", "pv_cell_mean", "conv3x3x3_tc", "trilinear_devoxelize"])
def test_launch_count_matches_profiled_kernels(case):
    from abi_cases import counted_and_traced
    from abi_cases_pvcnn import EXPECTED_KERNEL, LAUNCH_CASES
    call = LAUNCH_CASES[case][1]()
    torch.cuda.synchronize()
    for _ in range(3):          # a profiling session may come back without records; see tests/test_gpu_launch_count.py
        counted, names = counted_and_traced(call)
        if names:
            break
    assert names, "%s: no kernel activity in three profiling sessions (counter grew by %d)" % (case, counted)
    assert counted == len(names), (case, counted, names)
    k = EXPECTED_KERNEL[case]
    assert any(k + "<" in m or k + "(" in m for m in (n.replace(" ", "") for n in names)), names
