"""Neighbour-search benchmark: fixed_radius_search, radius_search (one radius per query), the L1 / Linf metrics,
knn_search with and without ignore_query_point, and layers.ContinuousConv with per-point extents and a window.

    python bench_search.py [--reps R]

Workloads (seeded): a 65 536-point synth.room_cloud searched against itself at the KPConv S3DIS level-0 radius 0.1
(fixed_radius_search L2 is the path KPFCNN runs; radius_search with every radius 0.1 must return the same rows bit
for bit; radii drawn from U(0.05, 0.15); L1 and Linf at 0.1); k = 16 nearest neighbours on a 45 056-point
synth.semantickitti_cloud against itself (L2, L1, and L2 with ignore_query_point); the ContinuousConv layer at the
shape bench_cconv_transpose.py uses (16 384 inputs, 65 536 outputs, filter [4, 4, 4, 64, 64]) with per-point extents
and a poly6 window.  Timed with CUDA events in steady state; every search includes its one device->host read.  Prints
one JSON line with the card's name, power limit and maximum SM clock, and writes nothing.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    from open3d_ml_b200 import layers as LY, ops, synth
    torch.cuda.set_device(0)
    room = synth.room_cloud(65536, 0)
    room = torch.from_numpy(room[0] if isinstance(room, tuple) else room).float().cuda().contiguous()
    kitti = torch.from_numpy(synth.semantickitti_cloud(45056, 0)).float().cuda().contiguous()
    g = torch.Generator().manual_seed(0)
    n = room.shape[0]
    const = torch.full((n,), 0.1, dtype=torch.float32, device="cuda")
    spread = (torch.rand(n, generator=g) * 0.1 + 0.05).cuda()

    fixed = ops.fixed_radius_search(room, room, 0.1)
    same = ops.radius_search(room, room, const, return_distances=True)
    rows_match = all(torch.equal(a, b) for a, b in zip(fixed, same))
    cases = {
        "fixed_radius_search_L2": lambda: ops.fixed_radius_search(room, room, 0.1),
        "radius_search_L2_const": lambda: ops.radius_search(room, room, const, return_distances=True),
        "radius_search_L2_spread": lambda: ops.radius_search(room, room, spread, return_distances=True),
        "fixed_radius_search_L1": lambda: ops.fixed_radius_search(room, room, 0.1, metric="L1"),
        "fixed_radius_search_Linf": lambda: ops.fixed_radius_search(room, room, 0.1, metric="Linf"),
        "knn16_L2": lambda: ops.knn_search(kitti, kitti, 16, return_distances=True),
        "knn16_L1": lambda: ops.knn_search(kitti, kitti, 16, metric="L1", return_distances=True),
        "knn16_L2_ignore": lambda: ops.knn_search(kitti, kitti, 16, ignore_query_point=True, return_distances=True),
    }
    entries = {"fixed_radius_search_L2": fixed.neighbors_index.numel(),
               "radius_search_L2_spread": cases["radius_search_L2_spread"]().neighbors_index.numel(),
               "fixed_radius_search_L1": cases["fixed_radius_search_L1"]().neighbors_index.numel(),
               "fixed_radius_search_Linf": cases["fixed_radius_search_Linf"]().neighbors_index.numel()}

    n_out, n_inp, cin, cout, nbrs = 65536, 16384, 64, 64, 32
    radius = (nbrs / (n_out * 4.0 / 3.0 * math.pi)) ** (1.0 / 3.0)
    out_pos, inp_pos = torch.rand(n_out, 3, generator=g).cuda(), torch.rand(n_inp, 3, generator=g).cuda()
    x = torch.randn(n_inp, cin, generator=g).cuda()
    ext = ((torch.rand(n_out, generator=g) * 0.5 + 0.75) * 2 * radius).cuda()
    layer = LY.ContinuousConv(cin, cout, [4, 4, 4], align_corners=True, coordinate_mapping="ball_to_cube_radial",
                              interpolation="linear", normalize=False,
                              window_function=lambda r2: torch.clamp((1 - r2) ** 3, 0, 1)).cuda().eval()
    with torch.no_grad():
        cases["continuous_conv_layer_per_point_poly6"] = lambda: layer(x, inp_pos, out_pos, ext)
        ms = {name: ev_time_ms(fn, args.reps, 3) for name, fn in cases.items()}
    print(json.dumps(dict(
        metric="neighbor_search", room_points=n, kitti_points=kitti.shape[0], radius=0.1, knn_k=16,
        radius_search_const_rows_equal_fixed=rows_match, neighbor_entries=entries,
        ms={k: round(v, 4) for k, v in ms.items()}, gpu=gpu_info(),
        timed="CUDA events, steady state, %d calls each after 3 warm-up calls; searches include their host read"
              % args.reps)))


if __name__ == "__main__":
    main()
