"""Records tests/golden/pvcnn_s3dis.manifest.json and boundary_pvcnn_class.npz from the UNMODIFIED reference PVCNN class
(through oracle/refshim.py, torch CPU; oracle/pvcnn.py binds the devoxelization rule the reference tree lacks) with
seeded weights on seeded, margin-nudged inputs.

    python tests/golden/make_golden_pvcnn.py

Needs the reference tree, like make_golden.py, whose seed and sampling it shares.  Inputs are not stored: they are pure
functions of the seeds (tests/pvcnn_support.py).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from oracle import refshim, weights, pvcnn as PV  # noqa: E402
import pvcnn_support as PS  # noqa: E402
from make_golden import SEED, sample_idx  # noqa: E402

PVCNN_CASES = dict(shipped=dict(width_multiplier=1, voxel_resolution_multiplier=2, seed0=500),
                   odd=dict(width_multiplier=0.5, voxel_resolution_multiplier=1.5, seed0=510))


def make_pvcnn():
    """The shipped S3DIS config and one with resolutions that are no powers of two (48 and 24) at half width, both on
    B = 2 margin-filtered room clouds of 4096 points: sampled logits and taps of the unmodified class."""
    ref = PV.bind_pvcnn_devoxelize()
    cfg = refshim.load_cfg("pvcnn_s3dis.yml")
    m = cfg.model.to_dict() if hasattr(cfg.model, "to_dict") else dict(cfg.model)
    B, N = 2, 4096
    save = dict(weight_seed=SEED, B=B, N=N)
    for tag, case in PVCNN_CASES.items():
        mc = dict(m, width_multiplier=case["width_multiplier"],
                  voxel_resolution_multiplier=case["voxel_resolution_multiplier"], device="cpu")
        net = ref.PVCNN(**mc)
        net.eval()
        man = weights.manifest_from_state_dict(net.state_dict())
        pcfg = dict(num_classes=mc["num_classes"], extra_feature_channels=mc["extra_feature_channels"],
                    width_multiplier=mc["width_multiplier"],
                    voxel_resolution_multiplier=mc["voxel_resolution_multiplier"])
        if tag == "shipped":
            weights.save_manifest(os.path.join(HERE, "pvcnn_s3dis.manifest.json"), man,
                                  dict(source="ml3d/configs/pvcnn_s3dis.yml", cfg=pcfg))
        sd = weights.seeded_state_dict(man, SEED)
        net.load_state_dict(sd, strict=True)
        inp = PS.pvcnn_inputs(B, N, case["seed0"], pcfg)
        taps, hooks = {}, []
        for i in range(4):
            blk = net.point_features[i]
            p = "point_features.%d" % i
            hooks.append(blk.voxelization.register_forward_hook(
                lambda mod, a, o, p=p: taps.__setitem__(p + ".voxels", o[0])))
            for j, li in enumerate((2, 5)):
                hooks.append(blk.voxel_layers[li].register_forward_hook(
                    lambda mod, a, o, p=p, j=j: taps.__setitem__("%s.conv%d" % (p, j), o.clone())))
            hooks.append(blk.register_forward_hook(lambda mod, a, o, p=p: taps.__setitem__(p, o[0].transpose(1, 2))))
        hooks.append(net.cloud_features.register_forward_hook(lambda mod, a, o: taps.__setitem__("cloud_features", o)))
        with torch.no_grad():
            out = net(inp)
        for h in hooks:
            h.remove()
        ptaps = {}
        with torch.no_grad():
            port = PV.pvcnn_forward(sd, inp, pcfg, taps=ptaps)
        err = (port - out).abs().max().item() / out.abs().max().item()
        print("pvcnn %s: port vs reference rel err %.3e" % (tag, err))
        assert err < 1e-5
        save[tag + ".cfg"] = json.dumps(dict(pcfg, seed0=case["seed0"]))
        save[tag + ".manifest"] = json.dumps(man)
        idx = sample_idx(out.numel(), 20000, 4)
        save[tag + ".logits_shape"] = np.array(out.shape)
        save[tag + ".logits_idx"], save[tag + ".logits"] = idx, out.reshape(-1)[idx].numpy()
        for k, v in taps.items():
            idx = sample_idx(v.numel(), 4096, 5)
            save["%s.tap.%s.idx" % (tag, k)] = idx
            save["%s.tap.%s" % (tag, k)] = v.reshape(-1)[idx].numpy()
            save["%s.tap.%s.max" % (tag, k)] = float(v.abs().max())
    np.savez_compressed(os.path.join(HERE, "boundary_pvcnn_class.npz"), **save)


if __name__ == "__main__":
    torch.set_num_threads(8)
    make_pvcnn()
