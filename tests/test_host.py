"""Host-side logic that needs no GPU: the open3d shim wiring, seeded generators,
frame sharding + the post-batch collectives over gloo (world_size 2)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import refshim, weights
from open3d_ml_b200 import synth, shard
import helpers as H


def test_synth_is_deterministic_and_in_range():
    a, b = synth.lidar_frame(5000, 9), synth.lidar_frame(5000, 9)
    assert np.array_equal(a, b) and a.dtype == np.float32 and a.shape == (5000, 4)
    r = synth.KITTI_RANGE
    assert (a[:, 0] >= r[0]).all() and (a[:, 0] < r[3]).all() and (a[:, 1] >= r[1]).all() and (a[:, 1] < r[4]).all()
    p, f = synth.room_cloud(3000, 1)
    assert p.shape == (3000, 3) and f.shape == (3000, 5)
    assert len(np.unique(np.round(p / 0.04).astype(np.int64), axis=0)) == 3000   # pre-gridded at dl


def test_seeded_weights_are_deterministic_and_nontrivial():
    sd1, _ = H.state_dict("randlanet_semantickitti.manifest.json", 5)
    sd2, _ = H.state_dict("randlanet_semantickitti.manifest.json", 5)
    sd3, _ = H.state_dict("randlanet_semantickitti.manifest.json", 6)
    assert all(torch.equal(sd1[k], sd2[k]) for k in sd1)
    assert not torch.equal(sd1["fc0.weight"], sd3["fc0.weight"])
    assert sd1["bn0.running_var"].min() >= 0.5 and sd1["decoder.0.conv.weight"].shape == (768, 256, 1, 1)


def test_shard_bounds_cover_everything_once():
    for n in (1, 7, 8, 32, 33):
        for w in (1, 2, 4, 8):
            seen = []
            for r in range(w):
                lo, hi = shard.shard_bounds(n, r, w)
                seen += list(range(lo, hi))
            assert seen == list(range(n))


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    n_frames = 5
    lo, hi = shard.shard_bounds(n_frames, rank, world)
    local = torch.stack([torch.full((6,), f, dtype=torch.int32) for f in range(lo, hi)]) if hi > lo \
        else torch.zeros((0, 6), dtype=torch.int32)
    allr = shard.gather_frame_results(local, n_frames)
    conf = torch.eye(3, dtype=torch.int64) * (rank + 1)
    shard.reduce_confusion(conf)
    q.put((rank, allr[:, 0].tolist(), conf.diag().tolist()))
    dist.destroy_process_group()


def test_frame_shard_collectives_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in procs)
    [p.join(60) for p in procs]
    for _, frames, diag in res:
        assert frames == [0, 1, 2, 3, 4] and diag == [3, 3, 3]


@pytest.mark.skipif(not refshim.available(), reason="/root/reference absent (GPU box)")
def test_shim_exposes_the_reference_tree_unmodified():
    """run in a subprocess: the shim owns sys.modules['open3d']"""
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from open3d_ml_b200 import shim; shim.install('/root/reference')\n"
            "import open3d as o3d, open3d.ml as _ml3d, open3d.ml.torch as ml3d\n"
            "from open3d.ml.torch.ops import voxelize, ragged_to_dense\n"
            "from open3d.ml.torch.layers import FixedRadiusSearch\n"
            "from open3d.ml.utils import Config as _C2\n"
            "from open3d.ml.torch.models import RandLANet as _R2\n"
            "import ml3d.utils as _mu; assert _C2 is _mu.Config\n"
            "import open3d.core as o3c\n"
            "assert o3d._build_config['BUILD_PYTORCH_OPS'] and o3c.nns.NearestNeighborSearch\n"
            "cfg = _ml3d.utils.Config.load_from_file('/root/reference/ml3d/configs/randlanet_semantickitti.yml')\n"
            "net = ml3d.models.RandLANet(**cfg.model)\n"
            "assert ml3d.pipelines.SemanticSegmentation and ml3d.models.PointPillars and ml3d.models.KPFCNN\n"
            "print('ok', sum(p.numel() for p in net.parameters()))\n") % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "ok 1242307" in r.stdout


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


def test_pipelined_runner_tree_helpers_and_cpu_refusal():
    """The pytree helpers of pipeline.py on CPU tensors, and the runner's refusal to exist without CUDA."""
    import torch
    from open3d_ml_b200 import pipeline as P
    host = dict(a=[torch.arange(6.).view(2, 3), torch.ones(4, dtype=torch.int64)], b=torch.zeros(2), n=7, z=None)
    dev = P._alloc_like(host, "cpu")
    assert P._same_layout(dev, host) and dev["n"] == 7 and dev["z"] is None
    assert dev["a"][0].shape == (2, 3) and dev["a"][1].dtype == torch.int64
    out = P._copy_tree(dev, host)
    assert torch.equal(out["a"][0], host["a"][0]) and torch.equal(out["a"][1], host["a"][1]) and out["n"] == 7
    other = dict(host, b=torch.zeros(3))
    assert not P._same_layout(dev, other)
    assert not P._same_layout(dev, dict(a=host["a"], b=host["b"], n=7))          # key set differs
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            P.PipelinedRunner(lambda x: x)


@pytest.mark.skipif(not refshim.available(), reason="/root/reference absent (GPU box)")
def test_reference_boundary_script_dry_run_with_oracle_ops():
    """tests/ref_boundary_cases.py (the script behind the -m gpu boundary tests) on this CPU box with the oracle
    bound instead of the CUDA library: the unmodified RandLANet preprocess / transform / forward flow works."""
    import json
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_boundary_cases.py"),
                        "randlanet_patch", "--ops", "oracle"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert res["ops"] == "oracle" and res["ref_shape"] == [1, 8192, 19]
