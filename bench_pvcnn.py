"""PVCNN at the shipped S3DIS config (pvcnn_s3dis.yml: 40 960 points, 9 channels, grids of 64^3 and 32^3).

    python bench_pvcnn.py [--reps R] [--warmup W] [--batches 1,4]

Per batch size (1 is the config's test batch): the fused forward replayed from its CUDA graph and launched eagerly, the
torch port of the reference (oracle/pvcnn.py) run eagerly on the same GPU with TF32 disabled for cuDNN and matmul
(the like-for-like precision) and with TF32 allowed (a lower-precision run), two alternating runs of each side; the
stages of the fused forward timed one by one with CUDA events on the forward's own buffers (cells, grouping, cell mean,
each of the eight convolutions, devoxelization, the 1344 -> 512 layer; "rest" is the eager forward minus their sum);
and, per convolution, the algorithmic flop of its shapes (2 per multiply-add, counted here) over its time, and that rate
against the H100 SXM data sheet's dense TF32 rate of 495 TFLOP/s.  The kernel issues three TF32 products per
algorithmic one (3xTF32), so a third of the data-sheet rate is the most the algorithmic rate can reach; the first
layer pads its 9 channels to 32 and issues 32 / 9 of its algorithmic products on top of that.  The outputs of both
sides are compared at the timed size.  Weights are seeded from tests/golden/pvcnn_s3dis.manifest.json, inputs are
synth.pvcnn_s3dis_input (seeds 700 + b) through oracle.pvcnn.pv_margin_nudge.  Prints one JSON line with the card's
name, power limit and max SM clock, and writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_pointpillars_configs import ev_time_ms, gpu_info  # noqa: E402

TF32_PEAK_TFLOPS = 495.0     # NVIDIA H100 SXM data sheet, dense TF32


def stage_times(net, inp, reps, warm):
    """CUDA-event times of the forward's stages, each launched alone over the buffers one forward left behind."""
    from open3d_ml_b200 import _lib as L
    from open3d_ml_b200.pvcnn import LEAKY, VOXEL_EPS, pad32
    net.forward(inp)
    B, _, N = inp["point"].shape
    buf, w = net.buf.get, net.w
    coords, cat = buf("coords", (B * N, 3)), buf("cat", (B * N, net.ccat))
    out = dict(cells=0.0, grouping=0.0, cell_mean=0.0, devoxelize=0.0, convs=[])
    groups = {}
    for r in sorted(set(net.res)):
        tag = "r%d." % r
        vox, cell, stats = buf(tag + "vox", (B * N, 3)), buf(tag + "cell", (B * N,), torch.int32), buf(tag + "stats", (B, 4))
        cells = ev_time_ms(lambda: L.check(L.lib().o3dml_pv_voxel_cells(
            L.ptr(coords), B, N, r, VOXEL_EPS, L.ptr(stats), L.ptr(vox), L.ptr(cell), L.stream())), reps, warm)
        both = ev_time_ms(lambda: groups.__setitem__(r, net.voxel_cells(coords, B, N, r)), reps, warm)
        out["cells"] += cells
        out["grouping"] += both - cells
    x, off = buf("feat", (B * N, net.in_channels)), 0
    for i, r in enumerate(net.res):
        p = "point_features.%d" % i
        vox, splits, ids = groups[r]
        cin, co, ncell = x.shape[1], net.widths[i], B * r ** 3
        g0 = buf("grid.in.%d.%d" % (r, pad32(cin)), (B, r, r, r, pad32(cin)))
        g1, g2 = buf("grid.a.%d.%d" % (r, co), (B, r, r, r, co)), buf("grid.b.%d.%d" % (r, co), (B, r, r, r, co))
        out["cell_mean"] += ev_time_ms(lambda: L.check(L.lib().o3dml_pv_cell_mean(
            L.ptr(splits), L.ptr(ids), ncell, L.ptr(x), x.stride(0), cin, pad32(cin), L.ptr(g0), L.stream())), reps, warm)
        for j, (src, dst, ci) in enumerate(((g0, g1, cin), (g1, g2, co))):
            ms = ev_time_ms(lambda: L.conv3x3x3(src, w["%s.conv%d.wt" % (p, j)], dst, w["%s.conv%d.s" % (p, j)],
                                                w["%s.conv%d.t" % (p, j)], "leaky", LEAKY), reps, warm)
            flop = 2.0 * 27 * ci * co * ncell
            out["convs"].append(dict(layer="%s.conv%d" % (p, j), grid=r, cin=ci, cout=co, ms=round(ms, 4),
                                     algorithmic_gflop=round(flop / 1e9, 2),
                                     issued_over_algorithmic=round(3.0 * pad32(ci) / ci, 2),
                                     algorithmic_tflops=round(flop / ms / 1e9, 2),
                                     share_of_tf32_data_sheet=round(flop / ms / 1e9 / TF32_PEAK_TFLOPS, 4)))
        # timed writing, not accumulating: the buffer it adds to would otherwise grow from launch to launch
        scratch = buf("bench.devox", (B * N, co))
        out["devoxelize"] += ev_time_ms(lambda: L.check(L.lib().o3dml_trilinear_devoxelize(
            L.ptr(vox), B, N, r, L.ptr(g2), co, co, 0, L.ptr(scratch), co, None, None, L.stream())), reps, warm)
        x, off = cat[:, off:off + co], off + co
    c1 = w["classifier.0.wt"].shape[1]
    shift, h1 = buf("classifier.0.shift", (B, c1)), buf("classifier.0", (B * N, c1))

    def classifier0():
        for b in range(B):
            rows = slice(b * N, (b + 1) * N)
            net._lin("classifier.0", [L.make_src(cat[rows])], h1[rows], shift=shift[b])
    out["classifier_1344_512"] = ev_time_ms(classifier0, reps, warm)
    out["conv_sum"] = sum(c["ms"] for c in out["convs"])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", default="1,4")
    args = ap.parse_args()
    import open3d_ml_b200 as M
    from open3d_ml_b200 import synth
    from oracle import pvcnn as PV, weights
    if not torch.cuda.is_available():
        raise SystemExit("bench_pvcnn.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    man, extra = weights.load_manifest(os.path.join(ROOT, "tests", "golden", "pvcnn_s3dis.manifest.json"))
    sd, cfg = weights.seeded_state_dict(man, 1), extra["cfg"]
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    net = M.PVCNNB200(sd, cfg)
    n = 40960
    res = {}
    for B in [int(b) for b in args.batches.split(",")]:
        # points are kept 1e-3 of a voxel off the rounding boundaries, so that both sides voxelize alike
        clouds = [(PV.pv_margin_nudge(p, sorted(set(net.res))), f)
                  for p, f in (synth.pvcnn_s3dis_input(n, 700 + b) for b in range(B))]
        inp = dict(point=torch.from_numpy(np.stack([c[0].T for c in clouds])).cuda().contiguous(),
                   feat=torch.from_numpy(np.stack([c[1].T for c in clouds])).cuda().contiguous())

        def port():
            with torch.no_grad():
                return PV.pvcnn_forward(sd_dev, inp, cfg)

        def with_tf32(on, fn):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = on
            try:
                return fn()
            finally:
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        runs = dict(fused_graphed_ms=[], fused_eager_ms=[], port_fp32_ms=[], port_tf32_ms=[])
        for _ in range(2):                                   # the sides alternate
            runs["fused_graphed_ms"].append(ev_time_ms(lambda: net.forward_graphed(inp), args.reps, args.warmup))
            runs["port_fp32_ms"].append(with_tf32(False, lambda: ev_time_ms(port, args.reps, 2)))
            runs["fused_eager_ms"].append(ev_time_ms(lambda: net.forward(inp), args.reps, args.warmup))
            runs["port_tf32_ms"].append(with_tf32(True, lambda: ev_time_ms(port, args.reps, 2)))
        got, want = net.forward(inp), with_tf32(False, port)
        low = with_tf32(True, port)
        scale = float(want.abs().max())
        stages = stage_times(net, inp, args.reps, args.warmup)
        eager = min(runs["fused_eager_ms"])
        known = sum(stages[k] for k in ("cells", "grouping", "cell_mean", "devoxelize", "conv_sum", "classifier_1344_512"))
        stages["rest"] = eager - known
        res["B%d" % B] = dict(
            points=B * n, **{k: [round(v, 4) for v in vs] for k, vs in runs.items()},
            fused_vs_port_fp32_rel_err=float((got - want).abs().max()) / scale,
            port_tf32_vs_port_fp32_rel_err=float((low - want).abs().max()) / scale,
            argmax_agreement=float((got.argmax(-1) == want.argmax(-1)).float().mean()),
            stages_ms={k: (round(v, 4) if not isinstance(v, list) else v) for k, v in stages.items()})
    print(json.dumps(dict(metric="PVCNN S3DIS forward", config="ml3d/configs/pvcnn_s3dis.yml", results=res,
                          gpu=gpu_info(), tf32_data_sheet_tflops=TF32_PEAK_TFLOPS,
                          timed="CUDA events, steady state, x%d each after %d warm-up calls (torch port: after 2); "
                                "each side run twice, alternating" % (args.reps, args.warmup))))


if __name__ == "__main__":
    main()
