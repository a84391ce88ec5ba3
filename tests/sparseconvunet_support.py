"""The recorded SparseConvUnet cases of tests/golden/boundary_sparseconvunet_class.npz (make_golden_sparseconvunet.py):
the seeded state_dict, the config, the batch the reference's preprocess / transform / ConcatBatcher built, and the
logits of the unmodified class.  Importing this module needs no GPU."""
import json
import os
import types

import numpy as np
import torch

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "boundary_sparseconvunet_class.npz")
TAGS = ("shipped", "plain")


def recorded_case(tag):
    """-> (state_dict, cfg, batch with `point` / `feat` lists and `batch_lengths`, logits float32 [sum N, classes])."""
    from oracle import sparseconvunet as SP
    g = np.load(GOLDEN)
    cfg = json.loads(str(g[tag + ".cfg"]))
    sd = SP.seeded_state_dict(cfg, cfg.pop("weight_seed"))
    lengths = [int(x) for x in g[tag + ".lengths"]]
    splits = np.cumsum([0] + lengths)
    pts = g[tag + ".cells"].astype(np.float32) + np.float32(0.5)
    feat = g[tag + ".feat"]
    batch = types.SimpleNamespace(point=[torch.from_numpy(pts[a:b].copy()) for a, b in zip(splits[:-1], splits[1:])],
                                  feat=[torch.from_numpy(feat[a:b].copy()) for a, b in zip(splits[:-1], splits[1:])],
                                  batch_lengths=lengths)
    return sd, cfg, batch, torch.from_numpy(g[tag + ".logits"])


def rel_err(got, want):
    return float((got.double().cpu() - want.double()).abs().max() / want.abs().max())
