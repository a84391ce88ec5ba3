"""The instances of gemm_tc_kernel (open3d-ml_b200/csrc/gemm_tc.cu) and a Python copy of the rule in choose_instance that
picks one, so that tests/test_gpu_gemm_tc_matrix.py can derive from the SM count a shape that reaches each instance and
check from the profiler trace that it did.  Importing this module needs no GPU."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "open3d-ml_b200", "csrc")

ROWS, TILE_K, LITE_MAX_SLICES = 128, 32, 16      # GT_ROWS, GT_KS, GT_LITE_MAX_SLICES


def inst(bn, gather=False, lite=False, table=False, weighted=False):
    """An instance as its template argument list <BN, GATHER, LITE, TABLE, WEIGHTED>."""
    return (bn, gather, lite, table, weighted)


def inst_name(i):
    return "<%d, %s>" % (i[0], ", ".join("true" if b else "false" for b in i[1:]))


GATHER = {bn: inst(bn, gather=True) for bn in (32, 64, 128)}
LITE = {bn: inst(bn, lite=True) for bn in (32, 64)}
PLAIN = {bn: inst(bn) for bn in (32, 64, 128)}
MATRIX_INSTANCES = sorted([*GATHER.values(), *LITE.values(), *PLAIN.values()])
# table mode (the sparse convolutions): tests/test_gpu_sparse_contract.py and tests/test_gpu_sparse_weighted.py
TABLE_INSTANCES = sorted(inst(bn, True, False, True, w) for bn in (32, 64, 128) for w in (False, True))


def _arg(tok):
    tok = tok.strip()
    return {"true": True, "false": False}.get(tok, None if not tok.isdigit() else int(tok))


def launched_instances(path=os.path.join(CSRC, "gemm_tc.cu")):
    """The entries of GT_INSTANCES in gemm_tc.cu, the instances gemm_tc_launch dispatches to, as a sorted list with one
    entry per gt_entry<...>."""
    with open(path) as f:
        src = f.read()
    table = re.search(r"GT_INSTANCES\[\] = \{(.*?)\};", src, re.S)
    assert table, "no GT_INSTANCES list in " + path
    found = []
    for m in re.finditer(r"gt_entry<([^<>]*)>", table.group(1)):
        args = [_arg(t) for t in m.group(1).split(",")]
        assert len(args) == 5 and None not in args, "unparsed template arguments: " + m.group(0)
        found.append(inst(*args))
    return sorted(found)


def traced(call):
    """abi_cases.counted_and_traced, profiled again (up to five sessions) when a session delivers no activity records,
    as tests/test_gpu_launch_count.py does; in a long pytest process that has happened three times in a row.  The call
    must be safe to repeat."""
    from abi_cases import counted_and_traced
    for _ in range(5):
        counted, names = counted_and_traced(call)
        if names:
            break
    return counted, names


def traced_instance(names):
    """The template arguments of the gemm_tc_kernel activities in a profiler trace, e.g. from
    'void o3dml::gemm_tc_kernel<64, false, true, false, false>(o3dml::GemmTcParams)'."""
    out = []
    for n in names:
        m = re.search(r"gemm_tc_kernel<([^<>]*)>", n)
        if m:
            out.append(tuple(_arg(t) for t in m.group(1).split(",")))
    return out


def n_pad(cout):
    """_lib.PackedWeight's padding of the output channels: the weight image rows."""
    return 32 if cout <= 32 else 64 if cout <= 64 else (cout + 127) // 128 * 128


def ceil_div(a, b):
    return -(-a // b)


def conv3x3_tiles(H, W, stride):
    """128-pixel patches per image of a 3x3 convolution: the fewest over the patch shapes set_tiles tries."""
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    return min(ceil_div(OW, 1 << l) * ceil_div(OH, ROWS >> l) for l in range(8))


def conv3x3x3_tiles(X, Y, Z):
    """128-voxel boxes per grid of a 3x3x3 convolution: the fewest over the box shapes set_tiles tries."""
    return min(ceil_div(Z, 1 << lz) * ceil_div(Y, 1 << ly) * ceil_div(X, ROWS >> (lz + ly))
               for lz in range(8) for ly in range(8 - lz))


def route(row_tiles, cout, k, sms, rows_mode=True, gather=False):
    """choose_instance's choice for a product of `row_tiles` 128-row tiles, K = k, `cout` output columns, on `sms` SMs:
    the padded width is the tile width up to 64 and 128 beyond; short products of plain row sources that fill the SMs
    more than once run on the LITE kernels (64 columns at most); 128-column grids that fill at most half the SMs run as
    64-column tiles."""
    npad, kpad = n_pad(cout), ceil_div(k, TILE_K) * TILE_K
    bn = npad if npad <= 64 else 128
    lite = (rows_mode and not gather and kpad // TILE_K <= LITE_MAX_SLICES and
            row_tiles * (npad // (32 if bn == 32 else 64)) > sms)
    if lite and bn == 128:
        bn = 64
    if bn == 128 and 2 * row_tiles * (npad // 128) <= sms:
        bn = 64
    return inst(bn, gather, lite)
