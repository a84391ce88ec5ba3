"""The C-ABI shared library loads and exports every symbol include/o3dml_b200.h declares
(no compute calls: this runs without a GPU)."""
import ctypes
import os
import re

from conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "o3dml_b200.h")).read()
    return sorted(set(re.findall(r"O3DML_API[^;(]*?\b(o3dml_\w+)\s*\(", src)))


def test_header_declares_the_path():
    names = declared_symbols()
    for must in ("o3dml_voxelize", "o3dml_ragged_to_dense", "o3dml_knn_search", "o3dml_radius_count",
                 "o3dml_radius_fill", "o3dml_pp_pfn_scatter", "o3dml_linear", "o3dml_conv3x3_nhwc",
                 "o3dml_deconv_nhwc", "o3dml_randla_lfa_pool", "o3dml_gather_max", "o3dml_kpconv_gather"):
        assert must in names


def test_library_builds_loads_and_exports_everything():
    from open3d_ml_b200 import build, _lib
    path = build.build()
    h = ctypes.CDLL(path)
    for name in declared_symbols():
        assert hasattr(h, name), name
    assert set(_lib.EXPORTS) == set(declared_symbols())     # python binding covers the header
    assert _lib.lib().o3dml_abi_version() == _lib.ABI_VERSION == 2
    assert _lib.lib().o3dml_last_error() is not None


def test_sass_is_sm90a_only():
    import subprocess
    from open3d_ml_b200 import build
    out = subprocess.run(["cuobjdump", "-lelf", build.build()], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_ops_fail_loudly_without_cuda():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    import open3d_ml_b200 as m
    with pytest.raises(RuntimeError, match="no CPU path|no CUDA"):
        m.knn_search(torch.zeros(4, 3), torch.zeros(4, 3), 2)
    with pytest.raises(RuntimeError):
        m.RandLANetB200({})
