"""SparseConvUnet at the shipped ScanNet config (sparseconvunet_scannet.yml: 2 cm voxels, multiplier 32, residual
blocks, one repetition, grid 4096).

    python bench_sparseconvunet.py [--points N] [--reps R] [--warmup W] [--batches 1,4]

Inputs are synth.sparseconvunet_scannet_input rooms (N points each, sampled at 1 cm; seeds 900 + b); the voxel count
of every level is printed.  Per batch size, with CUDA events: the fused forward launched eagerly (two runs); the
pyramid and tables on their own; per level, one BN-ReLU-3^3 contraction (planes -> planes) on the level's own table as
one table-mode launch (o3dml_sparse_conv_tc) and, alternating with it, as the grouping it replaced (nine gathered
GEMMs of three cells each, L.make_src / L.linear, the BN-ReLU applied by a separate torch pass), with the algorithmic
rate of the first (2 flop per multiply-add of the non-empty table entries); and the head (BN-ReLU-Linear gathered per
point) on its own.  The convolutions inside the forward are not timed one by one.  The fused output is compared with
the float64 torch port (oracle/sparseconvunet.py, run on the same GPU); the port is the oracle, not a speed baseline,
and is not timed.  Weights are seeded (oracle.sparseconvunet.seeded_state_dict).  Prints one JSON line with the card's
name, power limit and max SM clock, and writes nothing.
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from bench_pointpillars_configs import ev_time_ms, gpu_info  # noqa: E402

CFG = dict(multiplier=32, conv_block_reps=1, residual_blocks=True, in_channels=3, num_classes=20, grid_size=4096)


def grouped_contraction(feat, table, w, out, pre):
    """The nine-launch path: cells three at a time as index operands, each group adding onto out through its residual."""
    from open3d_ml_b200 import _lib as L
    x = torch.relu(feat * pre[0] + pre[1])
    for gi, a in enumerate(range(0, 27, 3)):
        srcs = [L.make_src(x, index=table[:, c:], index_ld=27) for c in range(a, a + 3)]
        L.linear(srcs, w[gi], out, None, None, residual=out if gi else None, act=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=150000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", default="1,4")
    a = ap.parse_args()
    from open3d_ml_b200 import _lib as L, layers as LY, synth
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    from oracle import sparseconvunet as SP
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = SP.seeded_state_dict(CFG, 1)
    net = SparseConvUnetB200(sd, CFG)
    res = dict(gpu=gpu_info(), config="sparseconvunet_scannet", points_per_room=a.points, batches={})
    for B in [int(b) for b in a.batches.split(",")]:
        items = [synth.sparseconvunet_scannet_input(a.points, 900 + b) for b in range(B)]
        batch = types.SimpleNamespace(point=[torch.from_numpy(p).cuda() for p, _ in items],
                                      feat=[torch.from_numpy(f).cuda() for _, f in items],
                                      batch_lengths=[len(p) for p, _ in items])
        r = {}
        with torch.no_grad():
            fwd = lambda: net(batch)  # noqa: E731
            r["forward_ms"] = [ev_time_ms(fwd, a.reps, a.warmup) for _ in range(2)]
            pts = torch.cat(batch.point)
            splits = torch.tensor([0] + list(torch.tensor(batch.batch_lengths).cumsum(0).tolist())).cuda()
            lv, sizes, _ = net.pyramid(pts, splits)
            r["voxels_per_level"] = sizes
            r["pyramid_and_tables_ms"] = ev_time_ms(lambda: net.tables(*net.pyramid(pts, splits)[:2]), a.reps, a.warmup)
            sub = net.tables(lv, sizes)[0]
            levels = []
            for l, M in enumerate(sizes):
                c = net.planes[l]
                g = torch.Generator().manual_seed(l)
                feat = torch.randn(M, c, generator=g).cuda()
                w = torch.randn(27, c, c, generator=g) / (27 * c) ** 0.5
                pre = (torch.rand(c, generator=g).cuda() + 0.5, torch.randn(c, generator=g).cuda())
                packed = LY.pack_cells(w)
                groups = [L.pack_linear(w[i:i + 3].reshape(-1, c)) for i in range(0, 27, 3)]
                out_new, out_old = torch.empty(M, c).cuda(), torch.empty(M, c).cuda()
                new = lambda: LY.contract_cells(feat, sub[l], packed, out_new, pre=pre)  # noqa: E731
                old = lambda: grouped_contraction(feat, sub[l], groups, out_old, pre)  # noqa: E731
                tn, to = [], []
                for _ in range(2):
                    tn.append(ev_time_ms(new, a.reps, a.warmup))
                    to.append(ev_time_ms(old, a.reps, a.warmup))
                nnz = int((sub[l] < M).sum())
                agree = float((out_new - out_old).abs().max() / out_old.abs().max())
                levels.append(dict(level=l, voxels=M, channels=c, table_mode_ms=tn, nine_launch_ms=to,
                                   table_mode_tflops=2.0 * nnz * c * c / (min(tn) * 1e-3) / 1e12, agreement=agree))
            r["conv3x3x3_per_level"] = levels
            x0 = torch.randn(sizes[0], net.planes[0], generator=torch.Generator().manual_seed(9)).cuda()
            vop = torch.randint(0, sizes[0], (pts.shape[0], 1), dtype=torch.int32,
                                generator=torch.Generator().manual_seed(10)).cuda()
            logits = torch.empty(pts.shape[0], net.num_classes).cuda()
            r["head_ms"] = ev_time_ms(lambda: LY.contract_cells(x0, vop, net.w["head"], logits, net.w["head.bias"],
                                                                pre=(net.w["head.s"], net.w["head.t"])), a.reps, a.warmup)
            want = SP.sparseconvunet_forward(sd, batch, CFG, device="cuda")
            got = net(batch)
            r["agreement_vs_port"] = float((got.double() - want).abs().max() / want.abs().max())
        res["batches"][str(B)] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
