"""Seeded calls of the PVCNN entries of the C ABI (include/o3dml_b200_pvcnn.h) and their case tables, in the shape of
abi_cases.py: LAUNCH_CASES {case: (the C entry the case is meant to reach, builder of its call)} and EXPECTED_KERNEL.
tests/test_abi_pvcnn.py checks that the table covers every entry that header declares, so a new entry is added here.
None of these entries takes a workspace.  Importing this module needs no GPU."""
import torch

from open3d_ml_b200 import _lib as L
from abi_cases import rnd


def pv_inputs(B=2, N=500, r=6, seed=50):
    """Point rows of B clouds and their voxel coordinates and cell ids at resolution r, from o3dml_pv_voxel_cells."""
    pts = (torch.rand(B * N, 3, generator=torch.Generator().manual_seed(seed)) * 4).cuda()
    stats, vox = torch.empty(B, 4).cuda(), torch.empty(B * N, 3).cuda()
    cell = torch.empty(B * N, dtype=torch.int32).cuda()

    def call():
        return L.lib().o3dml_pv_voxel_cells(L.ptr(pts), B, N, r, 1e-6, L.ptr(stats), L.ptr(vox), L.ptr(cell),
                                            L.stream())
    return pts, vox, cell, call


def case_pv_cell_mean(B=2, N=500, r=6, C=9):
    _, _, cell, call = pv_inputs(B, N, r)
    L.check(call())
    order = torch.argsort(cell.long(), stable=True)
    ids = order.to(torch.int32)
    splits = torch.searchsorted(cell.long()[order].contiguous(), torch.arange(B * r ** 3 + 1).cuda()).contiguous()
    feat, grid = rnd(B * N, C, seed=51), torch.empty(B * r ** 3, 32).cuda()
    return lambda: L.lib().o3dml_pv_cell_mean(L.ptr(splits), L.ptr(ids), B * r ** 3, L.ptr(feat), C, C, 32,
                                              L.ptr(grid), L.stream())


def case_conv3x3x3():
    x, w = rnd(2, 5, 6, 7, 32, seed=52), rnd(27 * 32, 16, seed=53)
    weight, out = L.pack_linear(w), torch.empty(2, 5, 6, 7, 16).cuda()
    return lambda: L.conv3x3x3(x, weight, out, act="leaky", slope=0.1)


def case_trilinear_devoxelize(B=2, N=500, r=6, C=32):
    _, vox, _, call = pv_inputs(B, N, r)
    L.check(call())
    grid, out = rnd(B * r ** 3, C, seed=54), torch.zeros(B * N, C).cuda()
    inds, wgts = torch.empty(B, 8, N, dtype=torch.int32).cuda(), torch.empty(B, 8, N).cuda()
    return lambda: L.lib().o3dml_trilinear_devoxelize(L.ptr(vox), B, N, r, L.ptr(grid), C, C, 1, L.ptr(out), C,
                                                      L.ptr(inds), L.ptr(wgts), L.stream())


LAUNCH_CASES = {
    "pv_voxel_cells": ("o3dml_pv_voxel_cells", lambda: pv_inputs()[3]),
    "pv_cell_mean": ("o3dml_pv_cell_mean", case_pv_cell_mean),
    "conv3x3x3_tc": ("o3dml_conv3x3x3_ndhwc_tc", case_conv3x3x3),
    "trilinear_devoxelize": ("o3dml_trilinear_devoxelize", case_trilinear_devoxelize),
}

# the kernel a case is meant to reach; with the spaces of the trace's name removed, it is followed by "<" or "("
EXPECTED_KERNEL = {
    "pv_voxel_cells": "pv_point_cells_kernel", "pv_cell_mean": "pv_cell_mean_kernel",
    "conv3x3x3_tc": "gemm_tc_kernel", "trilinear_devoxelize": "pv_devoxelize_kernel",
}
