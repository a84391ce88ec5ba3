"""The cost of the per-entry weight of the sparse-convolution contraction (o3dml_sparse_conv_weighted_tc).

    python bench_sparse_weighted.py [--points N] [--reps R] [--warmup W] [--batch B]

1. Per level of SparseConvUnet's pyramid over B rooms (synth.sparseconvunet_scannet_input, seeds 900 + b, built as
   bench_sparseconvunet.py builds them): one BN-ReLU-3^3 contraction (planes -> planes) on the level's own table,
   unweighted (o3dml_sparse_conv_tc) against weighted (o3dml_sparse_conv_weighted_tc, weights uniform in [0.5, 1.5]),
   alternating, twice each.
2. The raw ops on one room's level-0 voxels (voxel units, centres k + 0.5): ragged lists from an L-infinity
   fixed_radius_search of radius 1.5 (the 27-neighbourhood, kernel index from the offset), inverted with
   invert_neighbors_list for the transposed op.  ops.sparse_conv without and with both importances (normalize on),
   and ops.sparse_conv_transpose with out_importance and neighbours' importance (inp_neighbors_importance_sum as the
   divisor), each as the table build (ops._sparse_table) and the contraction, timed apart and alternating.
Every arm is compared with float64 (max |error| / max |reference|).  CUDA events; prints one JSON line with the card's
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
from bench_sparseconvunet import CFG  # noqa: E402


def ref_table(feat, table, w, pre=None, weight=None):
    """float64 sum_c W_c^T (weight[:, c] * pre(feat[table[:, c]])), shadow ids reading zero."""
    x = feat.double()
    if pre is not None:
        x = torch.relu(x * pre[0].double() + pre[1].double())
    xp = torch.cat([x, x.new_zeros(1, x.shape[1])])
    t = table.long().clamp(max=x.shape[0])
    out = torch.zeros(table.shape[0], w.shape[2], dtype=torch.float64, device=feat.device)
    for c in range(table.shape[1]):
        g = xp[t[:, c]]
        if weight is not None:
            g = g * weight[:, c:c + 1].double()
        out += g @ w[c].to(feat.device).double()
    return out


def ref_ragged(feat, w, idx, kidx, rows, m, wt):
    """float64 out[r] = sum over the entries e of row r of wt_e W[k_e]^T f[idx_e]."""
    out = torch.zeros(m, w.shape[2], dtype=torch.float64, device=feat.device)
    f = feat.double()
    for c in range(w.shape[0]):
        sel = kidx == c
        out.index_add_(0, rows[sel], (wt[sel, None].double() * f[idx[sel].long()]) @ w[c].to(feat.device).double())
    return out


def dev(a, b):
    return float((a.double() - b).abs().max() / b.abs().max())


def alternate(arms, reps, warmup, rounds=2):
    """{name: [ms per round]} with the arms timed in turn, `rounds` times."""
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(ev_time_ms(fn, reps, warmup))
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=150000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    a = ap.parse_args()
    import open3d_ml_b200 as M
    from open3d_ml_b200 import layers as LY, ops, synth
    from open3d_ml_b200.sparseconvunet import SparseConvUnetB200
    from oracle import sparseconvunet as SP
    torch.backends.cuda.matmul.allow_tf32 = False
    net = SparseConvUnetB200(SP.seeded_state_dict(CFG, 1), CFG)
    res = dict(gpu=gpu_info(), config="sparseconvunet_scannet", points_per_room=a.points, rooms=a.batch)
    items = [synth.sparseconvunet_scannet_input(a.points, 900 + b) for b in range(a.batch)]
    batch = types.SimpleNamespace(point=[torch.from_numpy(p).cuda() for p, _ in items],
                                  batch_lengths=[len(p) for p, _ in items])
    with torch.no_grad():
        pts = torch.cat(batch.point)
        splits = torch.tensor([0] + list(torch.tensor(batch.batch_lengths).cumsum(0).tolist())).cuda()
        lv, sizes, _ = net.pyramid(pts, splits)
        sub = net.tables(lv, sizes)[0]
        levels = []
        for l, m in enumerate(sizes):
            c = net.planes[l]
            g = torch.Generator().manual_seed(l)
            feat = torch.randn(m, c, generator=g).cuda()
            w = torch.randn(27, c, c, generator=g) / (27 * c) ** 0.5
            pre = (torch.rand(c, generator=g).cuda() + 0.5, torch.randn(c, generator=g).cuda())
            wt = (torch.rand(m, 27, generator=g) + 0.5).cuda()
            packed = LY.pack_cells(w)
            out_u, out_w = torch.empty(m, c).cuda(), torch.empty(m, c).cuda()
            t = alternate({"unweighted": lambda: LY.contract_cells(feat, sub[l], packed, out_u, pre=pre),
                           "weighted": lambda: LY.contract_cells(feat, sub[l], packed, out_w, pre=pre,
                                                                 entry_weight=wt)}, a.reps, a.warmup)
            levels.append(dict(level=l, voxels=m, channels=c, unweighted_ms=t["unweighted"], weighted_ms=t["weighted"],
                               dev_unweighted=dev(out_u, ref_table(feat, sub[l], w, pre)),
                               dev_weighted=dev(out_w, ref_table(feat, sub[l], w, pre, wt))))
        res["contraction_per_level"] = levels

        # the raw ops on room 0's level-0 voxels, in voxel units
        cells = torch.unique(torch.floor(batch.point[0]).to(torch.int64), dim=0)      # the rooms are in voxel units
        pos = (cells.to(torch.float32) + 0.5).contiguous()
        n = pos.shape[0]
        r = ops.fixed_radius_search(pos, pos, 1.5, return_distances=False, metric="Linf")
        idx, rs = r.neighbors_index, r.neighbors_row_splits
        rows = torch.repeat_interleave(torch.arange(n, device=pos.device), rs[1:] - rs[:-1])
        d = torch.round(pos[idx.long()] - pos[rows]).to(torch.int64) + 1
        kidx = (d[:, 0] * 3 + d[:, 1]) * 3 + d[:, 2]
        e = idx.numel()
        cin, cout = 32, 32
        g = torch.Generator().manual_seed(20)
        feat = torch.randn(n, cin, generator=g).cuda()
        k = torch.randn(27, cin, cout, generator=g) / (27 * cin) ** 0.5
        iimp, nimp = (torch.rand(n, generator=g) + 0.5).cuda(), (torch.rand(e, generator=g) + 0.5).cuda()
        oimp = (torch.rand(n, generator=g) + 0.5).cuda()
        fa = LY.aligned_rows(feat)
        dv = feat.device

        def build(weight_fn, i=idx, kk=kidx, s=rs):
            return ops._sparse_table("bench", i, kk, s, 27, n, dv, weight_fn)
        plain_tab, _, reps, _, lens = build(None)
        w_tab = build(lambda _r: nimp * iimp[idx.long()])
        packed = LY.pack_cells(k.repeat(reps, 1, 1))
        out_p, out_i = torch.empty(n, cout).cuda(), torch.empty(n, cout).cuda()
        inv_k = ops.invert_neighbors_list(n, idx, rs, kidx)
        inv_w = ops.invert_neighbors_list(n, idx, rs, nimp)
        t_idx, t_k, t_nimp, t_rs = inv_k.neighbors_index, inv_k.neighbors_attributes, inv_w.neighbors_attributes, \
            inv_k.neighbors_row_splits
        t_rows = torch.repeat_interleave(torch.arange(n, device=dv), t_rs[1:] - t_rs[:-1])
        isum = torch.zeros(n, device=dv).index_add_(0, idx.long(), nimp * oimp[rows])
        s = torch.where(isum != 0, 1.0 / isum, torch.ones_like(isum))
        t_tab = build(lambda rr: t_nimp * s[t_idx.long()] * oimp[rr], t_idx, t_k, t_rs)
        t_packed = LY.pack_cells(k.repeat(t_tab[2], 1, 1))
        out_t = torch.empty(n, cout).cuda()
        t = alternate({
            "sparse_conv_table": lambda: build(None),
            "sparse_conv_contract": lambda: LY.contract_cells(fa, plain_tab, packed, out_p),
            "importance_table": lambda: build(lambda _r: nimp * iimp[idx.long()]),
            "importance_contract": lambda: LY.contract_cells(fa, w_tab[0], packed, out_i, entry_weight=w_tab[1]),
            "transpose_table": lambda: build(lambda rr: t_nimp * s[t_idx.long()] * oimp[rr], t_idx, t_k, t_rs),
            "transpose_contract": lambda: LY.contract_cells(fa, t_tab[0], t_packed, out_t, entry_weight=t_tab[1]),
        }, a.reps, a.warmup)
        ones = torch.ones(e, device=dv)
        ref_p = ref_ragged(feat, k, idx, kidx, rows, n, ones) / lens.clamp_min(1).double().unsqueeze(1)
        wi = nimp * iimp[idx.long()]
        n_o = torch.zeros(n, dtype=torch.float64, device=dv).index_add_(0, rows, wi.double())
        ref_i = ref_ragged(feat, k, idx, kidx, rows, n, wi) / torch.where(n_o != 0, n_o, 1.0).unsqueeze(1)
        ref_t = ref_ragged(feat, k, t_idx, t_k, t_rows, n, t_nimp * s[t_idx.long()] * oimp[t_rows])
        got_p = M.ops.sparse_conv(k, feat, torch.empty(0), idx, kidx, torch.empty(0), rs, True)
        got_i = M.ops.sparse_conv(k, feat, iimp, idx, kidx, nimp, rs, True)
        got_t = M.ops.sparse_conv_transpose(k, oimp, feat, torch.empty(0), isum, torch.empty(0), t_idx, t_k, t_nimp, t_rs,
                                            True)
        res["raw_ops"] = dict(points=n, entries=e, repeats=reps, channels=[cin, cout],
                              ms={key: v for key, v in t.items()},
                              dev_sparse_conv=dev(got_p, ref_p), dev_sparse_conv_importance=dev(got_i, ref_i),
                              dev_sparse_conv_transpose=dev(got_t, ref_t))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
