"""The weighted sparse-convolution entry of the C ABI (include/o3dml_b200_sparse_weighted.h), held to what
tests/test_abi.py holds the entries of o3dml_b200.h to: the library exports every declared symbol, the Python binding
covers exactly the header and no other header's entries, every entry is reached by a launch case, and none of them is
a sizing function or a capability query (no GPU needed).  tests/test_gpu_launch_count_sparse_weighted.py checks the
launch counter of each case on the GPU."""
import ctypes
import os
import re
import subprocess
import sys

from conftest import ROOT


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "o3dml_b200_sparse_weighted.h")).read()
    return sorted(set(re.findall(r"O3DML_API[^;(]*?\b(o3dml_\w+)\s*\(", src)))


def test_library_exports_and_binding_cover_the_header():
    from open3d_ml_b200 import build, _lib
    h = ctypes.CDLL(build.build())
    names = declared_symbols()
    assert names == ["o3dml_sparse_conv_weighted_tc"]
    for name in names:
        assert hasattr(h, name), name
    assert set(_lib.SPARSE_WEIGHTED_EXPORTS) == set(names)
    assert not set(_lib.SPARSE_WEIGHTED_EXPORTS) & (set(_lib.EXPORTS) | set(_lib.PVCNN_EXPORTS) |
                                                   set(_lib.SPARSECONVUNET_EXPORTS))
    assert _lib.lib().o3dml_abi_version() == _lib.ABI_VERSION == 2


def test_every_entry_has_a_launch_case_and_none_enqueues_nothing():
    from open3d_ml_b200 import _lib
    from abi_cases_sparse_weighted import EXPECTED_KERNEL, LAUNCH_CASES
    launched = {entry for entry, _ in LAUNCH_CASES.values()}
    assert launched == set(_lib.SPARSE_WEIGHTED_EXPORTS)
    assert not [n for n in _lib.SPARSE_WEIGHTED_EXPORTS if n.endswith(("_workspace_bytes", "_supported"))]
    assert set(EXPECTED_KERNEL) == set(LAUNCH_CASES)


def _run(code):
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr


def test_shim_resolves_sparse_conv_transpose_without_cuda():
    _run("import torch, open3d_ml_b200.shim as shim\n"
         "shim.install()\n"
         "from open3d.ml.torch.ops import sparse_conv, sparse_conv_transpose\n"
         "from open3d_ml_b200 import _lib, ops\n"
         "assert sparse_conv_transpose is ops.sparse_conv_transpose and sparse_conv is ops.sparse_conv\n"
         "assert _lib._lib is None and not torch.cuda.is_initialized()\n")


def test_shim_under_the_oracle_bindings_raises_when_called():
    _run("import open3d_ml_b200.shim as shim\n"
         "from oracle import refshim\n"
         "shim.install(bindings=refshim.BINDINGS)\n"
         "from open3d.ml.torch.ops import sparse_conv_transpose\n"
         "try:\n"
         "    sparse_conv_transpose()\n"
         "except NotImplementedError:\n"
         "    pass\n"
         "else:\n"
         "    raise SystemExit('sparse_conv_transpose did not raise')\n")
