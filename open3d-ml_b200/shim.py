"""The drop-in boundary: a minimal ``open3d`` package, fabricated in ``sys.modules``, whose
``open3d.ml.torch.{ops,layers}``, ``open3d.core.nns`` and friends resolve to this library,
and whose ``open3d.ml`` / ``open3d.ml.torch`` namespaces re-export the UNMODIFIED
Open3D-ML tree (``ml3d/``) found at ``$OPEN3D_ML_ROOT`` -- the mechanism documented at
README.md:313-314 / set_open3d_ml_root.sh:1-3 of the reference.  With it,

    import open3d_ml_b200.shim as shim; shim.install("/path/to/Open3D-ML")
    import open3d.ml.torch as ml3d          # as scripts/run_pipeline.py:12,97 does
    net = ml3d.models.RandLANet(**cfg.model)

runs the reference's models, dataloaders and pipelines with every native op on the
sm_90a kernels.  Symbols that the reference imports at module load but that are outside
the hot path (SURVEY.md Appendix B checklist) raise NotImplementedError when CALLED.
"""
import importlib
import os
import sys
import types


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    m.__dict__.update(attrs)
    sys.modules[name] = m
    parent, _, leaf = name.rpartition(".")
    if parent and parent in sys.modules:
        setattr(sys.modules[parent], leaf, m)
    return m


def _not_on_hot_path(symbol):
    def f(*a, **k):
        raise NotImplementedError(
            "open3d_ml_b200: '%s' is outside the accelerated hot path (SURVEY.md section 8)" % symbol)
    f.__name__ = symbol.rsplit(".", 1)[-1]
    return f


class _AddictDict(dict):
    """addict.Dict work-alike for ml3d/utils/config.py:9 when addict is not installed."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        for a in args:
            for k, v in dict(a or {}).items():
                self[k] = self._conv(v)
        for k, v in kwargs.items():
            self[k] = self._conv(v)

    @classmethod
    def _conv(cls, v):
        if isinstance(v, dict) and not isinstance(v, cls):
            return cls(v)
        if isinstance(v, (list, tuple)):
            return type(v)(cls._conv(x) for x in v)
        return v

    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        return self[k]

    def __setattr__(self, k, v):
        self[k] = self._conv(v)

    def __missing__(self, k):
        v = type(self)()
        self[k] = v
        return v

    def to_dict(self):
        return {k: (v.to_dict() if isinstance(v, _AddictDict) else v) for k, v in self.items()}

    def copy(self):
        return type(self)(self)


class _AliasFinder:
    """`from open3d.ml.utils import Config` / `import open3d.ml.torch.models` go through the import system,
    not through attribute access: resolve `open3d.ml.<x>` -> `ml3d.<x>` and `open3d.ml.torch.<x>` -> `ml3d.torch.<x>`
    and register the SAME module object under both names (the mechanism of README.md:313-314)."""

    FABRICATED = ("open3d.ml.torch.ops", "open3d.ml.torch.layers", "open3d.ml.contrib")

    def find_spec(self, name, path=None, target=None):
        if not name.startswith("open3d.ml.") or name.startswith(self.FABRICATED):
            return None
        real = "ml3d." + name[len("open3d.ml."):]
        try:
            mod = importlib.import_module(real)
        except ImportError:
            return None
        from importlib.machinery import ModuleSpec

        class _Loader:
            def create_module(self, spec):
                return mod

            def exec_module(self, module):
                pass
        return ModuleSpec(name, _Loader(), is_package=hasattr(mod, "__path__"))


_INSTALLED = False


def install(ml3d_root=None):
    """Registers the fabricated ``open3d`` package.  Idempotent.  Does not touch CUDA."""
    global _INSTALLED
    if _INSTALLED:
        return
    import torch
    from . import ops as O

    root = ml3d_root or os.environ.get("OPEN3D_ML_ROOT")
    if "open3d" in sys.modules and not getattr(sys.modules["open3d"], "_o3dml_b200_shim", False):
        raise RuntimeError("open3d_ml_b200.shim: a real `open3d` is already imported")
    _module("open3d", _o3dml_b200_shim=True, __version__="0.0+o3dml_b200",
            _build_config={"BUILD_PYTORCH_OPS": True, "BUILD_TENSORFLOW_OPS": False,
                           "BUILD_GUI": False, "BUILD_CUDA_MODULE": True})
    core = _module("open3d.core", Tensor=O._O3CTensor)
    # device_count() = 0 keeps the reference from importing the CUDA-only PointNet++/PVCNN ops
    # (pointnet2_utils.py:35-36, roipool3d_utils.py:3-4, pvcnn.py:13-14), which are off the path
    _module("open3d.core.cuda", device_count=lambda: 0)
    _module("open3d.core.nns", NearestNeighborSearch=O.NearestNeighborSearch)
    core.nns, core.cuda = sys.modules["open3d.core.nns"], sys.modules["open3d.core.cuda"]
    ml = _module("open3d.ml")
    mlt = _module("open3d.ml.torch")
    _module("open3d.ml.torch.ops", voxelize=O.voxelize, ragged_to_dense=O.ragged_to_dense,
            knn_search=O.knn_search, fixed_radius_search=O.fixed_radius_search, radius_search=O.radius_search,
            nms=O.nms,
            reduce_subarrays_sum=O.reduce_subarrays_sum,
            voxel_pooling=O.voxel_pooling,
            continuous_conv=O.continuous_conv, continuous_conv_transpose=O.continuous_conv_transpose,
            invert_neighbors_list=O.invert_neighbors_list, sparse_conv=O.sparse_conv)
    from . import layers as LY
    _module("open3d.ml.torch.layers", FixedRadiusSearch=O.FixedRadiusSearch, RadiusSearch=O.RadiusSearch,
            KNNSearch=O.KNNSearch,
            SparseConv=LY.SparseConv, SparseConvTranspose=LY.SparseConvTranspose,
            ContinuousConv=LY.ContinuousConv, ContinuousConvTranspose=LY.ContinuousConvTranspose)
    _module("open3d.ml.contrib", subsample=O.subsample, subsample_batch=O.subsample_batch,
            iou_bev_cpu=O.iou_bev, iou_bev_cuda=O.iou_bev, iou_3d_cpu=O.iou_3d, iou_3d_cuda=O.iou_3d)
    vis = _module("open3d.visualization")
    tb = _module("open3d.visualization.tensorboard_plugin")
    _module("open3d.visualization.tensorboard_plugin.summary")
    vis.tensorboard_plugin = tb
    for n in ("open3d.geometry", "open3d.utility", "open3d.io", "open3d.t", "open3d.t.io",
              "open3d.visualization.gui", "open3d.visualization.rendering"):
        _module(n)
    # third-party packages the reference imports at module load and this image lacks
    try:
        import addict  # noqa: F401
    except ImportError:
        _module("addict", Dict=_AddictDict)
    try:
        import matplotlib  # noqa: F401
    except ImportError:
        _module("matplotlib")
        _module("matplotlib.pyplot")
        _module("matplotlib.cm")
    if root:
        if not os.path.isdir(os.path.join(root, "ml3d")):
            raise RuntimeError("open3d_ml_b200.shim: no ml3d/ under %s" % root)
        if root not in sys.path:
            sys.path.insert(0, root)

        def lazy(prefix):
            def getter(attr):
                if attr.startswith("__"):
                    raise AttributeError(attr)
                return importlib.import_module(prefix + "." + attr)
            return getter
        sys.meta_path.insert(0, _AliasFinder())
        ml.__getattr__ = lazy("ml3d")              # open3d.ml.utils / datasets / vis / configs
        mlt_get = lazy("ml3d.torch")               # open3d.ml.torch.models / pipelines / ...

        def mlt_getattr(attr):
            if attr in ("ops", "layers"):
                return sys.modules["open3d.ml.torch." + attr]
            return mlt_get(attr)
        mlt.__getattr__ = mlt_getattr
    _INSTALLED = True
