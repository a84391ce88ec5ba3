"""oracle/refshim.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Makes the UNMODIFIED reference model code importable in this container (torch CPU only) so that it can be used
as the model-layer oracle and to generate the golden fixtures under tests/golden/ (SURVEY.md section 8c,
Appendix B).  The `open3d` package is the one open3d_ml_b200.shim fabricates, with the reference's third-party
native ops (`open3d.ml.torch.ops`, `open3d.core.nns`, ...) bound to the CPU oracle in oracle/ops.py by BINDINGS.
"""
import collections
import os

import numpy as np
import torch

from . import ops as O
from .make_ref_snapshot import live_root, ref_root


def available():
    """Whether the unmodified reference tree itself is present (not only its oracle/_ref snapshot)."""
    return live_root() is not None


class Tensor:
    def __init__(self, a):
        self.a = np.asarray(a)

    @staticmethod
    def from_numpy(a):
        return Tensor(a)

    def numpy(self):
        return self.a


class NearestNeighborSearch:
    """dataprocessing.py:99-103"""

    def __init__(self, pts):
        self.p = pts.numpy()

    def knn_index(self):
        return True

    def knn_search(self, q, k):
        i, d = O.np_knn(self.p, q.numpy(), k)
        return Tensor(i.astype(np.int64)), Tensor(d)


_V = collections.namedtuple("VoxelizeResult", "voxel_coords voxel_point_indices "
                            "voxel_point_row_splits voxel_batch_splits")


def voxelize(points, row_splits, voxel_size, points_range_min, points_range_max,
             max_points_per_voxel=2**62, max_voxels=2**62):
    r = O.c_voxelize(points.detach().cpu().numpy(), row_splits.cpu().numpy(),
                     voxel_size.numpy(), points_range_min.numpy(),
                     points_range_max.numpy(), max_points_per_voxel, max_voxels)
    return _V(*(torch.from_numpy(r[k]) for k in _V._fields))


def ragged_to_dense(values, row_splits, out_col_size, default_value):
    return torch.from_numpy(O.np_ragged_to_dense(values.numpy(), row_splits.numpy(),
                                                 int(out_col_size),
                                                 default_value.numpy()))


def nms(boxes, scores, thr):
    keep, _ = O.c_nms(boxes.detach().cpu().numpy(), scores.detach().cpu().numpy(), float(thr))
    return torch.from_numpy(keep).to(boxes.device)


_R = collections.namedtuple("FixedRadiusSearchResult",
                            "neighbors_index neighbors_row_splits neighbors_distance")


class FixedRadiusSearch:
    """kpconv.py:2021-2026 (rows ordered by (d2, idx), DESIGN.md)."""

    def __call__(self, points, queries, radius, points_row_splits, queries_row_splits):
        i, rs, d = O.c_radius(points.numpy(), queries.numpy(), radius,
                              points_row_splits.numpy(), queries_row_splits.numpy())
        return _R(torch.from_numpy(i), torch.from_numpy(rs), torch.from_numpy(d))


def subsample_batch(points, batches_len, features=None, classes=None, sampleDl=0.1,
                    method="barycenter", max_p=0, verbose=0):
    r = O.c_subsample_batch(points, batches_len, features, classes, sampleDl, max_p)
    if classes is not None:
        r = r[:-1] + (r[-1].astype(np.asarray(classes).dtype),)
    return r


def subsample(points, features=None, classes=None, sampleDl=0.1, verbose=0):
    r = subsample_batch(points, [len(points)], features, classes, sampleDl)
    out = (r[0],) + tuple(r[2:])
    return out[0] if len(out) == 1 else out


def _iou_bev(a, b):
    return O.c_iou_matrix(a, b, 0)


def _iou_3d(a, b):
    return O.c_iou_matrix(a, b, 1)


BINDINGS = {
    "open3d.core": dict(Tensor=Tensor),
    "open3d.core.nns": dict(NearestNeighborSearch=NearestNeighborSearch),
    "open3d.ml.torch.ops": dict(voxelize=voxelize, ragged_to_dense=ragged_to_dense, nms=nms),
    "open3d.ml.torch.layers": dict(FixedRadiusSearch=FixedRadiusSearch),
    "open3d.ml.contrib": dict(subsample=subsample, subsample_batch=subsample_batch,
                              iou_bev_cpu=_iou_bev, iou_bev_cuda=_iou_bev, iou_3d_cpu=_iou_3d, iou_3d_cuda=_iou_3d),
}


def install():
    """Idempotent.  After this, `import open3d.ml.torch` and `import ml3d.torch` work (reference code).
    -> the reference root."""
    from open3d_ml_b200 import shim
    root = ref_root()
    if root is None:
        raise RuntimeError("no reference tree (see oracle/make_ref_snapshot.py)")
    shim.install(root, BINDINGS)
    return root


def load_cfg(yml_name):
    """Reference config loader (ml3d/utils/config.py:210-241) on a shipped yml."""
    root = install()
    from ml3d.utils import Config
    return Config.load_from_file(os.path.join(root, "ml3d", "configs", yml_name))
