"""Every *_workspace_bytes returns exactly the bytes its entry point carves.  Each entry that takes a workspace is called
with none (NULL, 0 bytes) and NULL for every device pointer: it must refuse with status 2 before it enqueues anything,
and the "(N needed)" of its message must equal what the sizing function returns.  The rows, and the sizing function
each one checks, are abi_cases.REFUSAL_ROWS.  Needs no GPU."""
import re

import numpy as np
import pytest

from open3d_ml_b200 import _lib as L
from abi_cases import REFUSAL_ROWS

VOXEL_HOST = [np.full(3, v, np.float32) for v in (0.5, 0.0, 4.0)]      # voxel size, range min, range max
SPARSE_OFFSET, SPARSE_KERNEL = np.zeros(3, np.float32), np.full(3, 3, np.int32)
# A host address for the pointers an entry checks for NULL before its workspace.  The workspace refusal comes first,
# so it is never dereferenced.
HOST_WORD = np.zeros(1, np.int64)
NONNULL = HOST_WORD.ctypes.data


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


def sizing(row, *args):
    """What the sizing function of REFUSAL_ROWS[row] returns for args."""
    return getattr(L.lib(), REFUSAL_ROWS[row][0])(*args)


@pytest.mark.parametrize("n,batch", REFUSAL_ROWS["voxelize"][1])
def test_voxelize(n, batch):
    h = VOXEL_HOST
    got = refused(lambda: L.lib().o3dml_voxelize(None, n, 4, None, batch, h[0].ctypes.data, h[1].ctypes.data,
                                                 h[2].ctypes.data, 32, 1000, None, None, None, None, None, None, None, 0,
                                                 None))
    assert got == sizing("voxelize", n, batch)


@pytest.mark.parametrize("np_,nq,batch", REFUSAL_ROWS["knn_search"][1])
def test_knn_search(np_, nq, batch):
    got = refused(lambda: L.lib().o3dml_knn_search(None, np_, None, None, nq, None, batch, 8, None, 0, None, None, 0,
                                                   None))
    assert got == sizing("knn_search", np_, nq, batch)


@pytest.mark.parametrize("np_,nq,batch,k,ignore", REFUSAL_ROWS["knn_search_metric"][1])
def test_knn_search_metric(np_, nq, batch, k, ignore):
    """ignore_query_point needs out_row_splits, which is checked first."""
    got = refused(lambda: L.lib().o3dml_knn_search_metric(None, np_, None, None, nq, None, batch, k, 1, ignore, None, 1,
                                                          None, NONNULL if ignore else None, None, None, 0, None))
    assert got == sizing("knn_search_metric", np_, nq, batch, k, ignore)


@pytest.mark.parametrize("np_,nq,batch", REFUSAL_ROWS["radius_count_and_fill"][1])
def test_radius_count_and_fill(np_, nq, batch):
    wsb = sizing("radius_count_and_fill", np_, nq, batch)
    assert refused(lambda: L.lib().o3dml_radius_count(None, np_, None, None, nq, None, batch, 0.8, None, None, None,
                                                      0, None)) == wsb
    assert refused(lambda: L.lib().o3dml_radius_fill(None, np_, nq, None, batch, 0.8, None, None, None, None, 0,
                                                     None)) == wsb


@pytest.mark.parametrize("np_,nq,batch", REFUSAL_ROWS["radius_search_count_and_fill"][1])
def test_radius_search_count_and_fill(np_, nq, batch):
    """One radius per query (radii non-NULL), L-infinity, ignore_query_point, normalize_distances, int64 ids."""
    wsb = sizing("radius_search_count_and_fill", np_, nq, batch)
    assert refused(lambda: L.lib().o3dml_radius_search_count(None, np_, None, None, nq, None, batch, 0.0, NONNULL, 2, 1,
                                                             None, None, None, 0, None)) == wsb
    assert refused(lambda: L.lib().o3dml_radius_search_fill(None, np_, nq, None, batch, 0.0, NONNULL, 2, 1, 1, None,
                                                            None, 1, None, None, 0, None)) == wsb


@pytest.mark.parametrize("num_entries", REFUSAL_ROWS["invert_neighbors_list"][1])
def test_invert_neighbors_list(num_entries):
    """Its input and output pointers are checked first."""
    got = refused(lambda: L.lib().o3dml_invert_neighbors_list(3000, NONNULL, 0, NONNULL, max(1, num_entries // 4),
                                                              num_entries, NONNULL, NONNULL, NONNULL, None, 0, None))
    assert got == sizing("invert_neighbors_list", num_entries)


@pytest.mark.parametrize("n", REFUSAL_ROWS["nms"][1])
def test_nms(n):
    got = refused(lambda: L.lib().o3dml_nms(None, None, n, 0.5, None, None, None, 0, None))
    assert got == sizing("nms", n)


@pytest.mark.parametrize("num_in,num_out", REFUSAL_ROWS["sparse_conv_neighbors"][1])
def test_sparse_conv_neighbors(num_in, num_out):
    got = refused(lambda: L.lib().o3dml_sparse_conv_neighbors(None, num_in, None, num_out, 1.0,
                                                              SPARSE_OFFSET.ctypes.data, SPARSE_KERNEL.ctypes.data, 0,
                                                              None, None, None, 0, None))
    assert got == sizing("sparse_conv_neighbors", num_in)


@pytest.mark.parametrize("B,H,W,A,C,nms_pre", REFUSAL_ROWS["pp_detect"][1])
def test_pp_detect(B, H, W, A, C, nms_pre):
    got = refused(lambda: L.lib().o3dml_pp_detect(None, 0, None, 0, None, 0, B, H, W, A, C, None, nms_pre, 0.1, 0.78,
                                                  None, None, None, None, None, 0, None))
    assert got == sizing("pp_detect", B, H, W, A, C, nms_pre)
