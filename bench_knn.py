"""k-NN benchmark for any k: knn_search past the 64 neighbours a row of the register kernel holds.

    python bench_knn.py [--reps R]

Workloads (seeded): a 45 056-point synth.semantickitti_cloud (RandLA-Net's SemanticKITTI input size) queried against
itself at k = 64 (knn_kernel<64>, for reference) and at k = 65, 128, 256 and 1024 (knn_select_kernel) in L2, plus L1 at
k = 128; and the reference's scene crop, search_tree.query(center_point, k=num_points): 8 queries with k = 45 056 on a
120 000-point cloud.  Each shape is also timed as a user would write it without this library, torch.cdist +
torch.topk(largest=False); that baseline is for timing only (its distances are not the contract's float32 order and
its ties are not ordered by index).  Timed with CUDA events in steady state, each search including its host read.
Prints one JSON line with the card's name, power limit and maximum SM clock, and writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench_detect import ev_time_ms, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_knn.py: needs a CUDA device")
    from open3d_ml_b200 import ops, synth
    torch.cuda.set_device(0)
    kitti = torch.from_numpy(synth.semantickitti_cloud(45056, 0)[:, :3]).float().cuda().contiguous()
    scene = torch.from_numpy(synth.semantickitti_cloud(120000, 1)[:, :3]).float().cuda().contiguous()
    g = torch.Generator().manual_seed(0)
    centres = scene[torch.randperm(scene.shape[0], generator=g)[:8].cuda()].contiguous()
    crop_k = 45056

    def ours(q, p, k, metric="L2"):
        return lambda: ops.knn_search(p, q, k, metric=metric, index_dtype=torch.int64, return_distances=True)

    def baseline(q, p, k, metric="L2"):
        return lambda: torch.topk(torch.cdist(q, p, p=2.0 if metric == "L2" else 1.0), k, dim=1, largest=False)

    shapes = {"self_k64_L2": (kitti, kitti, 64, "L2")}
    shapes.update({"self_k%d_L2" % k: (kitti, kitti, k, "L2") for k in (65, 128, 256, 1024)})
    shapes["self_k128_L1"] = (kitti, kitti, 128, "L1")
    shapes["crop_8q_k45056_L2"] = (centres, scene, crop_k, "L2")

    r64, r65 = ours(kitti, kitti, 64)(), ours(kitti, kitti, 65)()
    continues = torch.equal(r65.neighbors_index.view(-1, 65)[:, :64], r64.neighbors_index.view(-1, 64))
    ms = {name: ev_time_ms(ours(*s), args.reps, 2) for name, s in shapes.items()}
    base_ms = {name: ev_time_ms(baseline(*s), args.reps, 2) for name, s in shapes.items()}
    print(json.dumps(dict(
        metric="knn_any_k", kitti_points=kitti.shape[0], crop_points=scene.shape[0], crop_queries=centres.shape[0],
        crop_k=crop_k, k65_rows_continue_k64=continues,
        ms={k: round(v, 4) for k, v in ms.items()},
        baseline_cdist_topk_ms={k: round(v, 4) for k, v in base_ms.items()}, gpu=gpu_info(),
        timed="CUDA events, steady state, %d calls each after 2 warm-up calls; knn_search includes its host read"
              % args.reps)))


if __name__ == "__main__":
    main()
