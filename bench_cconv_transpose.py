"""Transposed continuous convolution benchmark: the steps of layers.ContinuousConvTranspose, and the forward op on the
mirrored graph for comparison.

    python bench_cconv_transpose.py [--reps R]

Workload: seeded clouds uniform in the unit cube, 65 536 output points (fine) and 16 384 input points (coarse); the
radius (extent / 2) is chosen so that an interior input has 32 output neighbours on average; filter [4, 4, 4, 64, 64],
linear interpolation, ball_to_cube_radial, align_corners.  Timed with CUDA events in steady state: the radius search,
invert_neighbors_list, continuous_conv_transpose, continuous_conv over the same entries with the input and output
roles swapped (the same kernel doing the same work), and the layer end to end.  The algorithmic rate of both
convolutions is 8 * 2 * Cin * Cout FLOP per neighbour entry (eight trilinear corners, one FMA per filter weight),
reported as a share of the H100 SXM data-sheet FP32 rate.  Prints one JSON line and writes nothing.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench_detect import ev_time_ms, gpu_info  # noqa: E402

FP32_PEAK_TFLOPS = 67.0       # H100 SXM data sheet, dense FP32, at up to 700 W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    from open3d_ml_b200 import layers as LY, ops
    torch.cuda.set_device(0)
    n_out, n_inp, cin, cout, nbrs = 65536, 16384, 64, 64, 32
    radius = (nbrs / (n_out * 4.0 / 3.0 * math.pi)) ** (1.0 / 3.0)
    ext = torch.tensor([2 * radius], dtype=torch.float32)
    g = torch.Generator().manual_seed(0)
    out_pos, inp_pos = torch.rand(n_out, 3, generator=g).cuda(), torch.rand(n_inp, 3, generator=g).cuda()
    x, y = torch.randn(n_inp, cin, generator=g).cuda(), torch.randn(n_out, cout, generator=g).cuda()
    layer = LY.ContinuousConvTranspose(cin, cout, [4, 4, 4], align_corners=True, coordinate_mapping="ball_to_cube_radial",
                                       interpolation="linear", normalize=False).cuda().eval()
    w = layer.kernel.detach()
    w_t = w.transpose(-1, -2).contiguous()
    off, empty = torch.zeros(3), torch.empty(0, device="cuda")
    cc = dict(align_corners=True, coordinate_mapping="ball_to_cube_radial", interpolation="linear")

    def search():
        return ops.fixed_radius_search(out_pos, inp_pos, float(ext[0]) * 0.5, return_distances=False)

    r = search()
    entries = int(r.neighbors_index.numel())

    def invert():
        return ops.invert_neighbors_list(n_out, r.neighbors_index, r.neighbors_row_splits, empty)

    inv = invert()

    def transpose():
        return ops.continuous_conv_transpose(w, out_pos, empty, ext, off, inp_pos, x, r.neighbors_index, empty,
                                             r.neighbors_row_splits, inv.neighbors_index, empty,
                                             inv.neighbors_row_splits, normalize=False, **cc)

    def forward_mirrored():
        return ops.continuous_conv(w_t, inp_pos, ext, off, out_pos, y, empty, r.neighbors_index, empty,
                                   r.neighbors_row_splits, normalize=False, **cc)

    with torch.no_grad():
        def layer_e2e():
            return layer(x, inp_pos, out_pos, ext)
        ms = {name: ev_time_ms(fn, args.reps, 5) for name, fn in
              (("radius_search", search), ("invert_neighbors_list", invert), ("continuous_conv_transpose", transpose),
               ("continuous_conv_mirrored", forward_mirrored), ("layer", layer_e2e))}
        # the two convolutions are adjoint: <forward(y), x> = <y, transpose(x)>, up to fp32 rounding
        a, b = (forward_mirrored().double() * x.double()).sum(), (y.double() * transpose().double()).sum()
        adjoint_rel = float((a - b).abs() / ((forward_mirrored() * x).abs().sum().double() + 1e-30))
    flop = entries * 8 * 2 * cin * cout
    rate = {k: flop / (ms[k] * 1e-3) / 1e12 for k in ("continuous_conv_transpose", "continuous_conv_mirrored")}
    print(json.dumps(dict(
        metric="continuous_conv_transpose", out_points=n_out, inp_points=n_inp, filter=[4, 4, 4, cin, cout],
        radius=round(radius, 6), neighbor_entries=entries, mean_neighbors_per_input=round(entries / n_inp, 2),
        ms={k: round(v, 4) for k, v in ms.items()},
        tflops={k: round(v, 3) for k, v in rate.items()},
        fp32_peak_share={k: round(v / FP32_PEAK_TFLOPS, 4) for k, v in rate.items()},
        adjoint_rel_gap=adjoint_rel, gpu=gpu_info(),
        timed="CUDA events, steady state, %d calls each after 5 warm-up calls; the search and the layer include the "
              "search's one host read" % args.reps)))


if __name__ == "__main__":
    main()
