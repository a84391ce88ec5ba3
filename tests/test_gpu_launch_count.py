"""o3dml_launch_count() against the kernels the GPU actually ran.  For every C-ABI entry, on a small valid input prepared
beforehand, one call is run under torch.profiler: the counter must grow by exactly the number of kernel activities
the profiler records for that call (memsets and copies are not kernels and are not counted).  Where a case names them,
the call must also reach its kernel and enqueue exactly the number of kernels it promises: one per sparse contraction,
whatever the number of kernel cells.  bench.py's gpu_launches and the replay accounting of pipeline.graph_replay both
rest on this counter.  The cases are abi_cases.LAUNCH_CASES, EXPECTED_LAUNCHES and EXPECTED_KERNEL; this is the one
module that opens profiling sessions."""
import pytest
import torch

from abi_cases import EXPECTED_KERNEL, EXPECTED_LAUNCHES, LAUNCH_CASES, counted_and_traced

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(LAUNCH_CASES))
def test_launch_count_matches_profiled_kernels(case):
    call = LAUNCH_CASES[case][1]()
    torch.cuda.synchronize()
    # Every case enqueues at least one kernel.  In a long pytest process a profiling session now and then comes back
    # with no activity records at all (the CUPTI buffers of that session were not delivered); such a session says
    # nothing about the counter, so the same call is profiled again.  A trace that holds records is always compared.
    for _ in range(3):
        counted, names = counted_and_traced(call)
        if names:
            break
    assert names, "%s: no kernel activity in three profiling sessions (counter grew by %d)" % (case, counted)
    assert counted == len(names), "%s: o3dml_launch_count grew by %d, the profiler saw %d kernels: %s" % (
        case, counted, len(names), names)
    if case in EXPECTED_LAUNCHES:
        assert counted == EXPECTED_LAUNCHES[case], "%s: %d kernels, expected %d: %s" % (
            case, counted, EXPECTED_LAUNCHES[case], names)
    if case in EXPECTED_KERNEL:
        k = EXPECTED_KERNEL[case]
        assert any(k + "<" in m or k + "(" in m for m in (n.replace(" ", "") for n in names)), names
