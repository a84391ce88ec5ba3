"""o3dml_launch_count() against the kernels the GPU actually ran, for the weighted sparse-convolution entry
(abi_cases_sparse_weighted.LAUNCH_CASES): one launch per contraction, whatever the number of kernel cells.  The module
is named to run right after tests/test_gpu_launch_count_pvcnn.py, so that all profiling sessions of a test process
follow one another."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cells,pre", [(27, True), (27, False), (8, True), (8, False), (1, True), (1, False)])
def test_one_launch_per_weighted_contraction(cells, pre):
    from abi_cases import counted_and_traced
    from abi_cases_sparse_weighted import EXPECTED_KERNEL, case_sparse_conv_weighted_tc
    call = case_sparse_conv_weighted_tc(cells=cells, pre=pre)
    torch.cuda.synchronize()
    for _ in range(3):          # a profiling session may come back without records; see tests/test_gpu_launch_count.py
        counted, names = counted_and_traced(call)
        if names:
            break
    assert names, "no kernel activity in three profiling sessions (counter grew by %d)" % counted
    assert counted == len(names) == 1, (counted, names)
    k = EXPECTED_KERNEL["sparse_conv_weighted_tc"]
    assert any(k + "<" in m or k + "(" in m for m in (n.replace(" ", "") for n in names)), names
