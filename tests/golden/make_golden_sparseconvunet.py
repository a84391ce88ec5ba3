"""Records tests/golden/sparseconvunet_scannet.manifest.json and boundary_sparseconvunet_class.npz from the UNMODIFIED
reference SparseConvUnet class (through oracle/refshim.py, torch CPU; oracle/sparseconvunet.py binds SparseConv,
SparseConvTranspose and reduce_subarrays_sum to the CPU oracle) with seeded weights and randomised BN statistics.

    python tests/golden/make_golden_sparseconvunet.py

Inputs are built by the reference's own preprocess (test split) / transform / ConcatBatcher from synth.room_cloud
scenes with colours, and stored (voxel-centre points as int16 cells, colours as float32): preprocess places each scene
with the model's own RNG.  The logits are stored whole (the scenes are small).  Needs the reference tree.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import refshim, weights, sparseconvunet as SP  # noqa: E402

# (config overrides, points per scene, room size in metres, scene seeds, weight seed).  Rooms of under a metre sampled
# at 1 cm: most 2 cm voxels hold several points and have neighbours in most of their 27 cells.
CASES = dict(shipped=(dict(), 3000, (0.8, 0.6, 0.5), (900, 901), 11),
             plain=(dict(multiplier=16, residual_blocks=False, conv_block_reps=2), 2000, (0.5, 0.5, 0.4), (902,), 12))


def make():
    ref = SP.bind_sparseconvunet()
    from open3d_ml_b200 import synth
    from ml3d.torch.dataloaders.concat_batcher import ConcatBatcher
    m = refshim.load_cfg("sparseconvunet_scannet.yml").model
    m = m.to_dict() if hasattr(m, "to_dict") else dict(m)
    save = {}
    for tag, (over, n, room, seeds, wseed) in CASES.items():
        mc = dict(m, **over)
        mc.pop("name", None)
        net = ref.SparseConvUnet(**dict(mc, device="cpu", seed=wseed))
        net.eval()
        cfg = dict(multiplier=mc["multiplier"], conv_block_reps=mc["conv_block_reps"],
                   residual_blocks=mc["residual_blocks"], in_channels=mc["in_channels"],
                   num_classes=mc["num_classes"], grid_size=mc["grid_size"])
        sd = SP.seeded_state_dict(cfg, wseed)
        net.load_state_dict(sd, strict=True)          # the reference's keys and shapes, exactly
        if tag == "shipped":
            weights.save_manifest(os.path.join(HERE, "sparseconvunet_scannet.manifest.json"),
                                  weights.manifest_from_state_dict(net.state_dict()),
                                  dict(source="ml3d/configs/sparseconvunet_scannet.yml", cfg=cfg, weight_seed=wseed))
        items = []
        for s in seeds:
            pts, f = synth.room_cloud(n, s, dl=0.01, room=room)
            d = net.preprocess(dict(point=pts, feat=f[:, 1:4] * 255.0, label=None), {"split": "test"})
            items.append({"data": net.transform(d, {}), "attr": {}})
        batch = ConcatBatcher("cpu", model="SparseConvUnet").collate_fn(items)["data"]
        with torch.no_grad():
            out = net(batch)
            port = SP.sparseconvunet_forward(sd, batch, cfg)
        err = float((port - out.double()).abs().max() / out.abs().max())
        print("sparseconvunet %s: %d points, %d level-0 voxels, port vs reference rel err %.3e"
              % (tag, out.shape[0], len(np.unique(np.floor(torch.cat(batch.point).numpy()), axis=0)), err))
        assert err < 1e-5
        save[tag + ".cfg"] = json.dumps(dict(cfg, weight_seed=wseed))
        save[tag + ".lengths"] = np.array(batch.batch_lengths)
        pts = torch.cat(batch.point).numpy()
        assert np.array_equal(np.floor(pts) + 0.5, pts) and pts.max() < 2 ** 15
        save[tag + ".cells"] = np.floor(pts).astype(np.int16)
        save[tag + ".feat"] = torch.cat(batch.feat).numpy().astype(np.float32)
        save[tag + ".logits"] = out.numpy().astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "boundary_sparseconvunet_class.npz"), **save)


if __name__ == "__main__":
    torch.set_num_threads(8)
    make()
