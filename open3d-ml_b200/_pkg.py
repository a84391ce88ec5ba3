"""Package body of open3d_ml_b200 (see open3d_ml_b200/__init__.py).

Hopper (sm_90a) operators behind the `open3d.ml.torch.ops` surface used by
Open3D-ML's PyTorch models, plus fused forwards for PointPillars, RandLA-Net and
KPFCNN.  Importing the package does not touch CUDA; calling any operator without the
CUDA library or a CUDA device raises RuntimeError (there is no CPU fallback).
"""
__version__ = "0.1.0"

from . import ops, synth, shard  # noqa: F401,E402
from .ops import (voxelize, ragged_to_dense, knn_search, fixed_radius_search,  # noqa: F401,E402
                  FixedRadiusSearch, KNNSearch, NearestNeighborSearch, subsample, subsample_batch,
                  nms, iou_bev, iou_3d)


def __getattr__(name):
    # model wrappers are imported lazily (they pull nothing heavy, but keep import light)
    if name in ("RandLANetB200",):
        from .randlanet import RandLANetB200
        return RandLANetB200
    if name in ("PointPillarsB200",):
        from .pointpillars import PointPillarsB200
        return PointPillarsB200
    if name in ("KPFCNNB200",):
        from .kpconv import KPFCNNB200
        return KPFCNNB200
    if name in ("PipelinedRunner",):
        from .pipeline import PipelinedRunner
        return PipelinedRunner
    raise AttributeError(name)
