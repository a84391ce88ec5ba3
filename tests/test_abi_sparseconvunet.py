"""The sparse-convolution entry of the C ABI (include/o3dml_b200_sparseconvunet.h), held to what tests/test_abi.py holds
the entries of o3dml_b200.h to: the library exports every declared symbol, the Python binding covers exactly the
header, every entry is reached by a launch case, and none of them is a sizing function or a capability query (no GPU
needed).  tests/test_gpu_launch_count_sparseconvunet.py checks the launch counter of each case on the GPU."""
import ctypes
import os
import re

from conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "o3dml_b200_sparseconvunet.h")).read()
    return sorted(set(re.findall(r"O3DML_API[^;(]*?\b(o3dml_\w+)\s*\(", src)))


def test_library_exports_and_binding_cover_the_header():
    from open3d_ml_b200 import build, _lib
    h = ctypes.CDLL(build.build())
    names = declared_symbols()
    assert names == ["o3dml_sparse_conv_tc"]
    for name in names:
        assert hasattr(h, name), name
    assert set(_lib.SPARSECONVUNET_EXPORTS) == set(names)
    assert not set(_lib.SPARSECONVUNET_EXPORTS) & (set(_lib.EXPORTS) | set(_lib.PVCNN_EXPORTS))
    assert _lib.lib().o3dml_abi_version() == _lib.ABI_VERSION == 2


def test_every_entry_has_a_launch_case_and_none_enqueues_nothing():
    from open3d_ml_b200 import _lib
    from abi_cases_sparseconvunet import EXPECTED_KERNEL, LAUNCH_CASES
    launched = {entry for entry, _ in LAUNCH_CASES.values()}
    assert launched == set(_lib.SPARSECONVUNET_EXPORTS)
    assert not [n for n in _lib.SPARSECONVUNET_EXPORTS if n.endswith(("_workspace_bytes", "_supported"))]
    assert set(EXPECTED_KERNEL) == set(LAUNCH_CASES)
