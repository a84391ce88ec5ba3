"""The fused SparseConvUnet forward (open3d_ml_b200.sparseconvunet) against the float64 torch port
(oracle/sparseconvunet.py) on synthetic ScanNet-like rooms: residual and plain blocks, multiplier 16 and 32, one and
two block repetitions, a batch holding a one-voxel item; the empty-cell trap (positive folded BN shifts around isolated
voxels); the refusals; one synchronising call per forward."""
import types
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def batch_of(items):
    return types.SimpleNamespace(point=[torch.from_numpy(p) for p, _ in items], feat=[torch.from_numpy(f) for _, f in items],
                                 batch_lengths=[len(p) for p, _ in items])


def run_both(cfg, items, seed=0, shift_bias=0.0):
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    from oracle import sparseconvunet as SP
    sd = SP.seeded_state_dict(cfg, seed, shift_bias)
    b = batch_of(items)
    with torch.no_grad():
        got = SparseConvUnetB200(sd, cfg)(b)
        want = SP.sparseconvunet_forward(sd, b, cfg, device="cuda")
    assert tuple(got.shape) == (sum(b.batch_lengths), cfg["num_classes"])
    return float((got.double() - want).abs().max() / want.abs().max())


CFG = dict(multiplier=32, conv_block_reps=1, residual_blocks=True, in_channels=3, num_classes=20, grid_size=4096)


@pytest.mark.parametrize("multiplier,reps,residual", [(32, 1, True), (16, 1, False), (16, 2, True), (32, 2, False)])
def test_matches_float64_port_on_rooms(multiplier, reps, residual):
    from open3d_ml_b200 import synth
    cfg = dict(CFG, multiplier=multiplier, conv_block_reps=reps, residual_blocks=residual)
    items = [synth.sparseconvunet_scannet_input(30000, 3), synth.sparseconvunet_scannet_input(12000, 4)]
    assert run_both(cfg, items, seed=multiplier + reps) < 1e-4


def test_batch_with_a_one_voxel_item():
    from open3d_ml_b200 import synth
    one = (np.full((5, 3), 17.5, np.float32), np.random.default_rng(0).random((5, 3)).astype(np.float32))
    items = [synth.sparseconvunet_scannet_input(8000, 5), one, synth.sparseconvunet_scannet_input(3000, 6)]
    assert run_both(dict(CFG, multiplier=16), items) < 1e-4


def test_empty_cells_contribute_zero_not_relu_of_bn_zero():
    """Isolated voxels (no neighbour at any level below the coarsest) and BN shifts pushed positive: relu(BN(0)) > 0 on
    every channel, so a contraction that let an empty cell through would be far off."""
    rng = np.random.default_rng(1)
    k = np.unique(rng.integers(0, 1000, (400, 3)) * 4, axis=0)[:300]
    pts = (k + 0.5).astype(np.float32)
    feat = rng.random((len(pts), 3)).astype(np.float32)
    assert run_both(dict(CFG, multiplier=16, residual_blocks=False), [(pts, feat)], shift_bias=1.0) < 1e-4


def test_refusals():
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200, patch_reference_model
    from oracle import sparseconvunet as SP
    cfg = dict(CFG, multiplier=16)
    sd = SP.seeded_state_dict(cfg, 0)
    with pytest.raises(RuntimeError, match="in_channels"):
        SparseConvUnetB200(sd, dict(cfg, in_channels=4))
    with pytest.raises(RuntimeError, match="multiplier"):
        SparseConvUnetB200(SP.seeded_state_dict(dict(cfg, multiplier=6), 0), dict(cfg, multiplier=6))
    bad = dict(sd)
    bad["unet.net.0.sub_sparse_conv1.net.offset"] = torch.full((3,), 0.5)
    with pytest.raises(RuntimeError, match="offset"):
        SparseConvUnetB200(bad, cfg)
    net = SparseConvUnetB200(sd, cfg)
    pts = np.array([[1.5, 2.5, 3.5], [4096.5, 1.5, 1.5]], np.float32)
    with pytest.raises(RuntimeError, match="outside"):
        with torch.no_grad():
            net(batch_of([(pts, np.ones((2, 3), np.float32))]))
    with pytest.raises(RuntimeError, match="outside"):
        with torch.no_grad():
            net(batch_of([(-pts[:1], np.ones((1, 3), np.float32))]))
    f = torch.ones(1, 3, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference-only"):
        net(types.SimpleNamespace(point=[torch.from_numpy(pts[:1])], feat=[f], batch_lengths=[1]))
    model = types.SimpleNamespace(state_dict=lambda: sd, cfg=cfg, training=True)
    patch_reference_model(model)
    with pytest.raises(RuntimeError, match="inference-only"):
        model.forward(batch_of([(pts[:1], np.ones((1, 3), np.float32))]))


def test_one_synchronising_call_per_forward():
    from open3d_ml_b200 import synth
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    from oracle import sparseconvunet as SP
    cfg = dict(CFG, multiplier=16)
    net = SparseConvUnetB200(SP.seeded_state_dict(cfg, 0), cfg)
    b = batch_of([synth.sparseconvunet_scannet_input(5000, 7), synth.sparseconvunet_scannet_input(4000, 8)])
    b.point = [p.cuda() for p in b.point]
    b.feat = [f.cuda() for f in b.feat]
    with torch.no_grad():
        net(b)                      # packs nothing new, but sizes the buffers
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("warn")
        try:
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                net(b)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [x for x in w if "synchroniz" in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]


@pytest.mark.parametrize("tag", ["shipped", "plain"])
def test_matches_recorded_reference_class(tag):
    """Against the logits of the unmodified reference class (tests/golden/make_golden_sparseconvunet.py): the shipped
    ScanNet config on a batch of two scenes, and plain blocks at multiplier 16 with two repetitions."""
    import sparseconvunet_support as SS
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    sd, cfg, batch, want = SS.recorded_case(tag)
    with torch.no_grad():
        got = SparseConvUnetB200(sd, cfg)(batch)
    assert tuple(got.shape) == tuple(want.shape)
    assert SS.rel_err(got, want) < 1e-4


def grid_edge_items():
    """Items whose voxels touch 0 and grid_size - 1 on every axis; along x, item b's last cell and item b + 1's first
    sit on the faces that meet across ITEM_SPACING."""
    rng = np.random.default_rng(5)
    g = CFG["grid_size"]
    items = []
    for i in range(3):
        corners = np.array([[x, y, z] for x in (0, 1, g - 2, g - 1) for y in (0, g - 1) for z in (0, 1, g - 1)])
        inner = rng.integers(0, 6, (300, 3)) + rng.choice([0, g - 6], (300, 3))
        k = np.concatenate([corners, inner])
        pts = (k + rng.random(k.shape) * 0.999).astype(np.float32)
        items.append((pts, rng.random((len(pts), 3)).astype(np.float32)))
    return items


def test_tables_at_grid_edges_match_the_lattice_rules():
    """tables(): the 3^3 tables against np_sub_table and the up / down links against np_parent_cell, per item, on every
    level, for items at the edges of the grid."""
    import torch
    from open3d_ml_b200.sparseconvunet import ITEM_SPACING, LEVELS, SparseConvUnetB200
    from oracle import sparseconvunet as SP
    cfg = dict(CFG, multiplier=16)
    net = SparseConvUnetB200(SP.seeded_state_dict(cfg, 0), cfg)
    items = grid_edge_items()
    pts = torch.cat([torch.from_numpy(p) for p, _ in items]).cuda()
    splits = torch.tensor([0] + list(np.cumsum([len(p) for p, _ in items]))).cuda()
    with torch.no_grad():
        lv, sizes, outside = net.pyramid(pts, splits)
        sub, down, up = net.tables(lv, sizes)
    assert outside == 0
    for l in range(LEVELS):
        k = lv[l][0][:sizes[l]].long().cpu().numpy()
        bid = lv[l][4][:sizes[l]].long().cpu().numpy()
        shifted = k + np.stack([bid * ITEM_SPACING, 0 * bid, 0 * bid], 1)
        assert np.array_equal(sub[l].cpu().numpy(), SP.np_sub_table(shifted)), l
        if l == 0:
            continue
        kf = lv[l - 1][0][:sizes[l - 1]].long().cpu().numpy()
        bf = lv[l - 1][4][:sizes[l - 1]].long().cpu().numpy()
        u = up[l].long().cpu().numpy()
        parent, cell = u // 8, u % 8
        _, _, want_cell = SP.np_parent_cell(kf)
        assert np.array_equal(cell, want_cell)
        assert np.array_equal(k[parent], kf // 2) and np.array_equal(bid[parent], bf)
        d = down[l].cpu().numpy()
        assert np.array_equal(d[parent, cell], np.arange(len(kf)))
        assert (d < len(kf)).sum() == len(kf)
    assert sizes[-1] >= 2 * len(items)          # the corners stay apart up to the coarsest level


def test_grid_edges_and_the_largest_batch_against_float64():
    from open3d_ml_b200.sparseconvunet import ITEM_SPACING, MAX_KEY
    cfg = dict(CFG, multiplier=16)
    assert run_both(cfg, grid_edge_items()) < 1e-4
    most = (MAX_KEY - cfg["grid_size"]) // ITEM_SPACING + 1
    assert most == 255
    rng = np.random.default_rng(6)
    one = [(rng.integers(0, cfg["grid_size"], (1, 3)).astype(np.float32) + 0.5, rng.random((1, 3)).astype(np.float32))
           for _ in range(most)]
    one[0] = (np.zeros((1, 3), np.float32), one[0][1])
    one[-1] = (np.full((1, 3), cfg["grid_size"] - 0.5, np.float32), one[-1][1])
    assert run_both(cfg, one) < 1e-4
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    from oracle import sparseconvunet as SP
    with pytest.raises(RuntimeError, match="items per batch"):
        with torch.no_grad():
            SparseConvUnetB200(SP.seeded_state_dict(cfg, 0), cfg)(batch_of(one + one[:1]))
