"""Seeded calls of the weighted sparse-convolution entry of the C ABI (include/o3dml_b200_sparse_weighted.h), in the
shape of abi_cases.py: LAUNCH_CASES {case: (the C entry the case is meant to reach, builder of its call)} and
EXPECTED_KERNEL.  tests/test_abi_sparse_weighted.py checks that the table covers every entry that header declares.
Importing this module needs no GPU."""
import torch

from open3d_ml_b200 import layers as LY
from abi_cases import rnd


def case_sparse_conv_weighted_tc(m=300, n=250, cin=48, cout=40, cells=27, pre=True):
    """One weighted contraction over a seeded table with shadow entries, with or without the BN-ReLU prologue."""
    g = torch.Generator().manual_seed(70)
    table = torch.randint(0, n + n // 3, (m, cells), generator=g, dtype=torch.int32).cuda()
    weight = torch.randn(m, cells, generator=g).cuda()
    feat, w = rnd(n, cin, seed=71), rnd(cells, cin, cout, seed=72)
    s, t = (rnd(cin, seed=73), rnd(cin, seed=74)) if pre else (None, None)
    packed, out = LY.pack_cells(w.cpu()), torch.empty(m, cout).cuda()
    return lambda: LY.contract_cells(feat, table, packed, out, pre=(s, t) if pre else None, entry_weight=weight)


LAUNCH_CASES = {
    "sparse_conv_weighted_tc": ("o3dml_sparse_conv_weighted_tc", case_sparse_conv_weighted_tc),
}

# the kernel a case is meant to reach; with the spaces of the trace's name removed, it is followed by "<" or "("
EXPECTED_KERNEL = {"sparse_conv_weighted_tc": "gemm_tc_kernel"}
