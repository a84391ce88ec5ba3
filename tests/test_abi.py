"""The C-ABI shared library loads and exports every symbol include/o3dml_b200.h declares, and the binding reads every
declaration of the headers (no compute calls: this runs without a GPU)."""
import ctypes
import re

import pytest


def declared_symbols(header="o3dml_b200.h"):
    """Every declaration of the header in order, a name declared twice listed twice."""
    from open3d_ml_b200 import _lib
    return [name for name, _, _ in _lib.declarations(_lib.read_header(header))]


def test_binding_parser_skips_nothing():
    """Every O3DML_API token of the two headers, but the one in its own #define, starts a prototype the binding
    parses; the product and bring-up headers share no name; a type without a ctypes type or a declaration the
    parser cannot read raises."""
    from open3d_ml_b200 import _lib
    names = {}
    for header in ("o3dml_b200.h", "o3dml_b200_bringup.h"):
        tokens = sum(len(re.findall(r"\bO3DML_API\b", line)) for line in _lib.read_header(header).splitlines()
                     if not line.strip().startswith("#define O3DML_API "))
        names[header] = declared_symbols(header)
        assert tokens == len(names[header]) > 0, header
    shared = set(names["o3dml_b200.h"]) & set(names["o3dml_b200_bringup.h"])
    assert not shared, "declared in both headers: %s" % ", ".join(sorted(shared))
    with pytest.raises(ValueError, match="no ctypes type"):
        _lib.declarations("/* a type without a mapping */\nO3DML_API int o3dml_x(const float* a,\n"
                          "                         double b, void* stream);\n")
    with pytest.raises(ValueError, match="cannot read"):
        _lib.declarations("O3DML_API int o3dml_x(int (*cb)(int));")


def test_header_declares_the_path():
    names = declared_symbols()
    for must in ("o3dml_voxelize", "o3dml_ragged_to_dense", "o3dml_knn_search", "o3dml_radius_count",
                 "o3dml_radius_fill", "o3dml_pp_pfn_scatter", "o3dml_linear", "o3dml_conv3x3_nhwc",
                 "o3dml_deconv_nhwc", "o3dml_randla_lfa_pool", "o3dml_gather_max", "o3dml_kpconv_gather",
                 "o3dml_sparse_conv_tc", "o3dml_sparse_conv_weighted_tc", "o3dml_pv_voxel_cells", "o3dml_pv_cell_mean",
                 "o3dml_conv3x3x3_ndhwc_tc", "o3dml_trilinear_devoxelize"):
        assert must in names
    twice = sorted({n for n in names if names.count(n) > 1})
    assert not twice, "declared more than once: %s" % ", ".join(twice)


def test_library_builds_loads_and_exports_everything():
    from open3d_ml_b200 import build, _lib
    path = build.build()
    h = ctypes.CDLL(path)
    for name in declared_symbols():
        assert hasattr(h, name), name
    assert _lib.EXPORTS == tuple(declared_symbols())     # python binding covers the header
    assert _lib.lib().o3dml_abi_version() == _lib.ABI_VERSION == 2
    assert _lib.lib().o3dml_last_error() is not None


# the exports that enqueue nothing: version, error and counter functions, sizing functions and capability queries
ENQUEUE_NOTHING = (
    "o3dml_abi_version", "o3dml_last_error", "o3dml_launch_count", "o3dml_launch_count_add",
    "o3dml_voxelize_workspace_bytes", "o3dml_knn_workspace_bytes", "o3dml_radius_workspace_bytes",
    "o3dml_knn_search_metric_workspace_bytes", "o3dml_sparse_conv_workspace_bytes",
    "o3dml_invert_neighbors_list_workspace_bytes", "o3dml_nms_workspace_bytes", "o3dml_pp_detect_workspace_bytes",
    "o3dml_linear_tc_supported", "o3dml_linear_rows_small_supported", "o3dml_randla_tail_supported",
)


def test_contract_tables_cover_every_export():
    """Every export is reached by a launch-count case or enqueues nothing, every expected kernel or launch count belongs
    to a launch-count case, and every sizing function is checked by an exact-workspace case on the GPU and by a refusal
    row without one."""
    from open3d_ml_b200 import _lib
    from abi_cases import EXPECTED_KERNEL, EXPECTED_LAUNCHES, LAUNCH_CASES, REFUSAL_ROWS, WORKSPACE_CASES
    exports, quiet = set(_lib.EXPORTS), set(ENQUEUE_NOTHING)
    launched = {entry for entry, _ in LAUNCH_CASES.values()}
    sizing = {name for name in exports if name.endswith("_workspace_bytes")}
    for what, names in [("not a launch case", (set(EXPECTED_KERNEL) | set(EXPECTED_LAUNCHES)) - set(LAUNCH_CASES)),
                        ("not exported", (launched | quiet) - exports),
                        ("both launched and enqueuing nothing", launched & quiet),
                        ("no launch-count case", exports - launched - quiet),
                        ("no exact-workspace case", sizing - {s for s, _ in WORKSPACE_CASES.values()}),
                        ("no refusal row", sizing - {s for s, _ in REFUSAL_ROWS.values()})]:
        assert not names, "%s: %s" % (what, ", ".join(sorted(names)))


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
