"""Every *_workspace_bytes returns exactly the bytes its entry point carves.  Each entry that takes a workspace is called
with none (NULL, 0 bytes) and NULL for every device pointer: it must refuse with status 2 before it enqueues anything,
and the "(N needed)" of its message must equal what the sizing function returns.  Needs no GPU."""
import re

import numpy as np
import pytest

from open3d_ml_b200 import _lib as L

VOXEL_HOST = [np.full(3, v, np.float32) for v in (0.5, 0.0, 4.0)]      # voxel size, range min, range max
SPARSE_OFFSET, SPARSE_KERNEL = np.zeros(3, np.float32), np.full(3, 3, np.int32)


def needed(rc):
    """The bytes a refused call says it needed."""
    msg = L.lib().o3dml_last_error().decode()
    assert rc == 2, msg
    m = re.search(r"workspace too small \((\d+) needed\)", msg)
    assert m, msg
    return int(m.group(1))


def refused(call):
    n0 = L.lib().o3dml_launch_count()
    got = needed(call())
    assert L.lib().o3dml_launch_count() == n0
    return got


@pytest.mark.parametrize("n,batch", [(1, 1), (500, 2), (40000, 3)])
def test_voxelize(n, batch):
    h = VOXEL_HOST
    got = refused(lambda: L.lib().o3dml_voxelize(None, n, 4, None, batch, h[0].ctypes.data, h[1].ctypes.data,
                                                 h[2].ctypes.data, 32, 1000, None, None, None, None, None, None, None, 0,
                                                 None))
    assert got == L.lib().o3dml_voxelize_workspace_bytes(n, batch)


@pytest.mark.parametrize("np_,nq,batch", [(0, 1, 1), (500, 300, 1), (6000, 5000, 3)])
def test_knn_search(np_, nq, batch):
    got = refused(lambda: L.lib().o3dml_knn_search(None, np_, None, None, nq, None, batch, 8, None, 0, None, None, 0,
                                                   None))
    assert got == L.lib().o3dml_knn_workspace_bytes(np_, nq, batch)


@pytest.mark.parametrize("np_,nq,batch", [(1, 1, 1), (400, 200, 2), (6000, 5000, 3)])
def test_radius_count_and_fill(np_, nq, batch):
    wsb = L.lib().o3dml_radius_workspace_bytes(np_, nq, batch)
    assert refused(lambda: L.lib().o3dml_radius_count(None, np_, None, None, nq, None, batch, 0.8, None, None, None,
                                                      0, None)) == wsb
    assert refused(lambda: L.lib().o3dml_radius_fill(None, np_, nq, None, batch, 0.8, None, None, None, None, 0,
                                                     None)) == wsb


@pytest.mark.parametrize("n", [1, 64, 65, 3000])
def test_nms(n):
    got = refused(lambda: L.lib().o3dml_nms(None, None, n, 0.5, None, None, None, 0, None))
    assert got == L.lib().o3dml_nms_workspace_bytes(n)


@pytest.mark.parametrize("num_in,num_out", [(0, 1), (1, 1), (200, 100), (5000, 100)])
def test_sparse_conv_neighbors(num_in, num_out):
    got = refused(lambda: L.lib().o3dml_sparse_conv_neighbors(None, num_in, None, num_out, 1.0,
                                                              SPARSE_OFFSET.ctypes.data, SPARSE_KERNEL.ctypes.data, 0,
                                                              None, None, None, 0, None))
    assert got == L.lib().o3dml_sparse_conv_workspace_bytes(num_in)


@pytest.mark.parametrize("B,H,W,A,C,nms_pre", [(1, 6, 5, 2, 3, 100), (2, 6, 5, 2, 3, 20), (1, 248, 216, 2, 3, 100),
                                               (2, 200, 176, 4, 3, 4096)])
def test_pp_detect(B, H, W, A, C, nms_pre):
    got = refused(lambda: L.lib().o3dml_pp_detect(None, 0, None, 0, None, 0, B, H, W, A, C, None, nms_pre, 0.1, 0.78,
                                                  None, None, None, None, None, 0, None))
    assert got == L.lib().o3dml_pp_detect_workspace_bytes(B, H, W, A, C, nms_pre)
