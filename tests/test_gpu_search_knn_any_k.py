"""k-NN search for k > 64 (knn_select_kernel in grid.cu: one CTA per query, a radix select over the cells within
reach of the k-th distance) bit-equal to the oracles of oracle/search.py: the C brute force (c_search_knn) up to
k = 1000, the cKDTree + lexsort restatement (np_search_knn) beyond.  Indices, distances, padding and row lengths, in
every metric, with and without ignore_query_point, int32 and int64 ids, with and without distances; rows of up to
4096 keys are sorted in shared memory and longer ones in the workspace, and both sides of that switch are covered.
Then the C-ABI contract of o3dml_knn_search_metric at k > 64, and the open3d.core.nns drop-in at k = 100."""
import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import open3d_ml_b200 as M
from open3d_ml_b200 import _lib as L, synth
import search_edge_cases as E
from oracle import search as S
from oracle.make_ref_snapshot import ref_root

pytestmark = pytest.mark.gpu


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

METRICS = ["L2", "L1", "Linf"]
KS = (65, 100, 128, 257, 1000, 4096, 4097)
C_ORACLE_MAX_K = 1000          # the C oracle's k-buffer is O(n k) per query: np_search_knn beyond
SMEM_K = 4096                  # rows of more keys are sorted in the workspace
# (ids, with distances): every k runs through each
OUTPUT_FORMS = [(torch.int32, True), (torch.int64, True), (torch.int32, False), (torch.int64, False)]


def self_and_jittered(p, n_self, n_jitter, seed):
    """Queries: n_self points of the cloud itself (ignore_query_point skips them) and n_jitter points near others."""
    rng = np.random.default_rng(seed)
    q = np.concatenate([p[rng.choice(len(p), n_self, replace=False)],
                        p[rng.choice(len(p), n_jitter, replace=False)] + rng.normal(0, 0.05, (n_jitter, 3))])
    return np.ascontiguousarray(q, np.float32)


def single(p, q):
    p, q = np.ascontiguousarray(p, np.float32), np.ascontiguousarray(q, np.float32)
    return p, q, np.array([0, len(p)], np.int64), np.array([0, len(q)], np.int64)


def room():
    p = synth.room_cloud(2500, 1)[0][:, :3]
    return single(p, self_and_jittered(p, 150, 50, 1))


def kitti(n=3000, seed=2):
    p = synth.semantickitti_cloud(n, seed)[:, :3]
    return single(p, self_and_jittered(p, 150, 50, seed))


def lattice():
    """Integer lattice: equal distances everywhere, which rank by index."""
    g = np.arange(14, dtype=np.float32)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    rng = np.random.default_rng(3)
    q = np.concatenate([p[rng.choice(len(p), 120, replace=False)],
                        rng.integers(0, 14, (60, 3)) + np.float32(0.5), [[6.5, 6.5, 6.5], [-3, -3, -3]]])
    return single(p, q)


def identical():
    p = np.tile(np.float32([[1.5, -2.0, 0.25]]), (1500, 1))
    return single(p, np.float32([[1.5, -2.0, 0.25], [1.5, -2.0, 0.5], [0, 0, 0], [100, 100, 100]]))


def line():
    t = np.arange(3000, dtype=np.float32) * np.float32(0.01)
    p = np.stack([t, 2 * t, -t], 1)
    return single(p, np.concatenate([p[::25], p[::37] + np.float32([0.003, -0.002, 0.0]), [[-5, 0, 0], [60, 0, 0]]]))


def offset1e7():
    p = synth.semantickitti_cloud(3000, 4)[:, :3] + np.float32(1e7)
    return single(p, self_and_jittered(p, 150, 50, 4))


def edge_case(name):
    c = E.case(name)
    return c.points, c.queries, c.ps, c.qs


# nonfinite: NaN / +-inf coordinates in some points and queries; outside: queries far outside the support box;
# batch: 120 items, empty and one-point items among them, items without queries
CLOUDS = {"room": room, "kitti": kitti, "lattice": lattice, "identical": identical, "line": line,
          "offset1e7": offset1e7, "nonfinite": functools.partial(edge_case, "nonfinite"),
          "outside": functools.partial(edge_case, "outside"), "batch": functools.partial(edge_case, "batch")}


@functools.lru_cache(maxsize=None)
def cloud(name):
    return CLOUDS[name]()


@functools.lru_cache(maxsize=None)
def device_cloud(name):
    return tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in cloud(name))


@functools.lru_cache(maxsize=None)
def oracle(name, k, metric, ignore):
    p, q, ps, qs = cloud(name)
    search = S.c_search_knn if k <= C_ORACLE_MAX_K else S.np_search_knn
    return search(p, q, k, ps, qs, S.METRICS[metric], ignore)


def host_ids(t, n):
    a = t.cpu().numpy().astype(np.int64)
    bad = (a < -1) | (a >= n)
    assert not bad.any(), "ids out of range: %s" % np.unique(a[bad])[:8]
    return a


def check(res, ref, k, ignore, n, index_dtype, with_d, what):
    ref_idx, ref_d, ref_n = ref
    if ignore:
        keep = np.arange(k)[None, :] < ref_n[:, None]
        want_rs, want_idx, want_d = np.concatenate([[0], np.cumsum(ref_n)]), ref_idx[keep], ref_d[keep]
    else:
        want_rs, want_idx, want_d = np.arange(len(ref_n) + 1) * k, ref_idx.reshape(-1), ref_d.reshape(-1)
    assert res.neighbors_index.dtype == index_dtype and res.neighbors_index.is_cuda, what
    got = host_ids(res.neighbors_index, n)
    assert got.shape == want_idx.shape, what
    wrong = np.flatnonzero(got != want_idx)
    assert not len(wrong), "%s: %d ids differ, first at %d: %d for %d" % (what, len(wrong), wrong[0], got[wrong[0]],
                                                                           want_idx[wrong[0]])
    assert np.array_equal(res.neighbors_row_splits.cpu().numpy(), want_rs), what
    if with_d:
        assert np.array_equal(res.neighbors_distance.cpu().numpy(), want_d), what
    else:
        assert res.neighbors_distance.numel() == 0, what


def item_sizes(name):
    return np.diff(cloud(name)[2])


def run_and_check(name, k, metric, ignore):
    p, q, ps, qs = device_cloud(name)
    ref = oracle(name, k, metric, ignore)
    short = bool((item_sizes(name) < k).any())
    for index_dtype, with_d in OUTPUT_FORMS:
        res = M.ops.knn_search(p, q, k, ps, qs, index_dtype=index_dtype, metric=metric, ignore_query_point=ignore,
                               return_distances=with_d, allow_short=short)
        check(res, ref, k, ignore, len(p), index_dtype, with_d,
              "%s k=%d %s ignore=%s %s d=%s" % (name, k, metric, ignore, index_dtype, with_d))


@pytest.mark.parametrize("name", list(CLOUDS))
@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_bit_equal_to_oracle(name, metric, ignore):
    """Every k of KS and k equal to the largest item; items smaller than k give padded (or, with ignore, short)
    rows."""
    for k in sorted(set(KS) | {int(item_sizes(name).max())}):
        run_and_check(name, k, metric, ignore)


@functools.lru_cache(maxsize=None)
def big_cloud():
    p = synth.semantickitti_cloud(9000, 5)[:, :3]
    return single(p, self_and_jittered(p, 40, 24, 5))


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("ignore", [False, True])
def test_rows_sorted_in_the_workspace(metric, ignore):
    """k past SMEM_K: the row's keys are sorted in the workspace, in one full and one partial chunk (4097), in two
    full chunks (8192), and at the item size (9000)."""
    p, q, ps, qs = big_cloud()
    dp, dq, dps, dqs = (torch.from_numpy(a).cuda() for a in (p, q, ps, qs))
    for k in (SMEM_K, SMEM_K + 1, 2 * SMEM_K, len(p)):
        ref = S.np_search_knn(p, q, k, ps, qs, S.METRICS[metric], ignore)
        for index_dtype, with_d in OUTPUT_FORMS[:2]:
            res = M.ops.knn_search(dp, dq, k, dps, dqs, index_dtype=index_dtype, metric=metric,
                                   ignore_query_point=ignore, return_distances=with_d)
            check(res, ref, k, ignore, len(p), index_dtype, with_d, "k=%d %s ignore=%s" % (k, metric, ignore))



@pytest.mark.parametrize("name", ["kitti", "lattice", "nonfinite", "batch"])
@pytest.mark.parametrize("metric", METRICS)
def test_k65_continues_the_k64_row(name, metric):
    """The first 64 columns of a k = 65 row (knn_select_kernel) are the k = 64 row (knn_kernel<64>)."""
    p, q, ps, qs = device_cloud(name)
    short = bool((item_sizes(name) < 65).any())
    kw = dict(metric=metric, return_distances=True, index_dtype=torch.int64, allow_short=short)
    r64 = M.ops.knn_search(p, q, 64, ps, qs, **kw)
    r65 = M.ops.knn_search(p, q, 65, ps, qs, **kw)
    assert torch.equal(r65.neighbors_index.view(-1, 65)[:, :64], r64.neighbors_index.view(-1, 64))
    assert torch.equal(r65.neighbors_distance.view(-1, 65)[:, :64], r64.neighbors_distance.view(-1, 64))


def test_crop_shaped_query():
    """The reference's scene crop (search_tree.query(center_point, k=num_points)): 8 queries, k = 45 056, on 120 000
    points."""
    p = synth.semantickitti_cloud(120_000, 6)[:, :3]
    q = p[np.random.default_rng(6).choice(len(p), 8, replace=False)]
    p, q, ps, qs = single(p, q)
    k = 45_056
    res = M.ops.knn_search(torch.from_numpy(p).cuda(), torch.from_numpy(q).cuda(), k, index_dtype=torch.int64,
                           return_distances=True)
    check(res, S.np_search_knn(p, q, k, ps, qs), k, False, len(p), torch.int64, True, "crop")


# ------------------------------------------------------------------------------------------------ the C-ABI contract
HOST_WORD = np.zeros(1, np.int64)
NONNULL = HOST_WORD.ctypes.data        # a non-NULL out_row_splits: the refusals come before any access


def metric_case(k, ignore, np_=6000, nq=300):
    """o3dml_knn_search_metric in L1 with int64 ids, as (sizing args, run(ws, nbytes), check())."""
    p, q, ps, qs = kitti(np_, 7)
    q = q[:nq]
    qs = np.array([0, len(q)], np.int64)
    dp, dq, dps, dqs = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (p, q, ps, qs))
    idx, d = torch.empty(len(q) * k, dtype=torch.int64).cuda(), torch.empty(len(q) * k).cuda()
    rs, total = torch.empty(len(q) + 1, dtype=torch.int64).cuda(), torch.zeros(1, dtype=torch.int64).cuda()

    def run(ws, nbytes):
        return L.lib().o3dml_knn_search_metric(L.ptr(dp), len(p), L.ptr(dps), L.ptr(dq), len(q), L.ptr(dqs), 1, k, 1,
                                               ignore, L.ptr(idx), 1, L.ptr(d), L.ptr(rs), L.ptr(total), ws, nbytes,
                                               L.stream())

    def verify():
        ref_idx, ref_d, n = (S.c_search_knn if k <= C_ORACLE_MAX_K else S.np_search_knn)(p, q, k, ps, qs, 1, bool(ignore))
        if ignore:
            keep = np.arange(k)[None, :] < n[:, None]
            t = int(n.sum())
            assert int(total.item()) == t
            assert np.array_equal(rs.cpu().numpy(), np.concatenate([[0], np.cumsum(n)]))
            assert np.array_equal(idx[:t].cpu().numpy(), ref_idx[keep])
            assert np.array_equal(d[:t].cpu().numpy(), ref_d[keep])
        else:
            assert np.array_equal(idx.cpu().numpy(), ref_idx.reshape(-1))
            assert np.array_equal(d.cpu().numpy(), ref_d.reshape(-1))
    return (len(p), len(q), 1, k, ignore), run, verify


# Run in a process of its own, so that the trace holds this call alone: in a long pytest process a profiling session
# can lose the first kernel records it should hold.
LAUNCH_SCRIPT = r"""
import json
import sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import torch
import test_gpu_search_knn_any_k as T
from abi_cases import counted_and_traced
from open3d_ml_b200 import _lib as L
k, ignore = int(sys.argv[2]), int(sys.argv[3])
args, run, verify = T.metric_case(k, ignore)
wsb = L.lib().o3dml_knn_search_metric_workspace_bytes(*args)
ws = torch.empty(wsb, dtype=torch.uint8).cuda()
n0 = L.lib().o3dml_launch_count()
rc = run(L.ptr(ws), wsb - 1)
out = dict(wsb=wsb, short_rc=rc, short_msg=L.lib().o3dml_last_error().decode(),
           short_launches=L.lib().o3dml_launch_count() - n0)
out["counted"], out["names"] = counted_and_traced(lambda: run(L.ptr(ws), wsb))
verify()
print(json.dumps(out))
"""


@pytest.mark.parametrize("k", [65, 300, SMEM_K + 904])
@pytest.mark.parametrize("ignore", [0, 1])
def test_workspace_sizing_and_launches(k, ignore):
    """The sizing function's bytes suffice (the rows equal the oracle's) and one byte less is refused before anything
    is enqueued; the launch counter equals the kernels the trace shows, one of them knn_select_kernel."""
    r = subprocess.run([sys.executable, "-c", LAUNCH_SCRIPT, ROOT, str(k), str(ignore)], capture_output=True,
                       text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["short_rc"] == 2 and "(%d needed)" % out["wsb"] in out["short_msg"], out["short_msg"]
    assert out["short_launches"] == 0
    names = out["names"]
    assert out["counted"] == len(names), names
    flat = [x.replace(" ", "") for x in names]
    assert sum("knn_select_kernel<1,%s>" % ("true" if ignore else "false") in x for x in flat) == 1, names
    assert any("knn_compact_kernel" in x for x in flat) == bool(ignore), names


@pytest.mark.parametrize("nq,k,ignore,message", [
    (1 << 22, 1 << 11, 1, "the ragged row scan is uint32"),
    (1 << 31, 65, 0, "num_queries must be below 2^31"),
    (1 << 30, 1 << 30, 0, "the workspace size would overflow"),
])
def test_refusals(nq, k, ignore, message):
    """Refused with status 1 before anything is enqueued; the sizing function returns SIZE_MAX."""
    assert L.lib().o3dml_knn_search_metric_workspace_bytes(1000, nq, 1, k, ignore) == 2 ** 64 - 1
    n0 = L.lib().o3dml_launch_count()
    rc = L.lib().o3dml_knn_search_metric(None, 1000, None, None, nq, None, 1, k, 0, ignore, None, 0, None,
                                         NONNULL if ignore else None, None, None, 0, None)
    assert rc == 1 and message in L.lib().o3dml_last_error().decode()
    assert L.lib().o3dml_launch_count() == n0


def test_knn_search_raw_entry_keeps_its_limit():
    rc = L.lib().o3dml_knn_search(None, 1000, None, None, 10, None, 1, 65, None, 0, None, None, 0, None)
    assert rc == 1 and "k must be in 1..64" in L.lib().o3dml_last_error().decode()


# --------------------------------------------------------------------------------------------------- the drop-in
SHIM_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle.make_ref_snapshot import ref_root
from open3d_ml_b200 import shim
root = ref_root() if sys.argv[3] == "reference" else None
shim.install(root)
import open3d.core as o3c
pc = np.load(sys.argv[2])["pc"]
out = {}
idx, d = o3c.nns.NearestNeighborSearch(o3c.Tensor.from_numpy(pc)).knn_search(o3c.Tensor.from_numpy(pc[:500]), 100)
out["nns_idx"], out["nns_d"] = idx.numpy(), d.numpy()
if root is not None:
    from ml3d.datasets.utils import DataProcessing
    out["dp_idx"] = np.asarray(DataProcessing.knn_search(pc, pc, 100))
np.savez(sys.argv[2], pc=pc, **out)
"""


def shim_run(tmp_path, pc, with_reference):
    path = str(tmp_path / "knn.npz")
    np.savez(path, pc=pc)
    r = subprocess.run([sys.executable, "-c", SHIM_SCRIPT, ROOT, path, "reference" if with_reference else "bare"],
                       capture_output=True, text=True, timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(path)


def test_shim_nearest_neighbor_search_k100(tmp_path):
    """open3d.core.nns.NearestNeighborSearch(points).knn_search(queries, 100), which stopped at 'k must be in 1..64'."""
    pc = synth.semantickitti_cloud(45_056, 8)[:, :3]
    got = shim_run(tmp_path, pc, False)
    ref_idx, ref_d, _ = S.c_search_knn(pc, pc[:500], 100)
    assert np.array_equal(got["nns_idx"], ref_idx) and np.array_equal(got["nns_d"], ref_d)


@pytest.mark.skipif(ref_root() is None, reason="no reference tree or snapshot of it")
def test_reference_dataprocessing_knn_search_k100(tmp_path):
    """The reference's DataProcessing.knn_search(pc, pc, 100) (RandLANet.transform with num_neighbors = 100)."""
    pc = synth.semantickitti_cloud(45_056, 9)[:, :3]
    got = shim_run(tmp_path, pc, True)
    ref_idx, _, _ = S.np_search_knn(pc, pc, 100)
    assert np.array_equal(got["dp_idx"].astype(np.int64), ref_idx)
    assert np.array_equal(got["nns_idx"], ref_idx[:500])
