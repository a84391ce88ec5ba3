"""Fused dispatch for the reference model classes: after ``shim.install``,

    import open3d_ml_b200.fuse as fuse; fuse.fuse_reference_models()

makes every ``RandLANet``, ``PointPillars``, ``KPFCNN``, ``PVCNN`` and ``SparseConvUnet`` of
``open3d.ml.torch.models`` run its fused forward in eval mode, without a line in the user's script.  The fused
model follows the weights: it is built from the instance's ``state_dict()`` at the first eval call and built again
whenever a parameter or buffer changed since (``load_state_dict``, ``load_ckpt``, an optimiser step, ``.to()``), so
the reference pipelines, which call ``model.eval()`` before they load a checkpoint, run the weights they loaded.
PointPillars' ``bbox_head.get_bboxes`` decodes on the device after a fused forward.  Train mode runs the reference
forward and ``get_bboxes`` untouched.  A config the fused path refuses logs one warning and keeps the
reference forward.

``patch`` is the other way in, behind each model module's ``patch_reference_model``: it switches one instance to a
fused model built once, a snapshot of the weights it holds then.
"""
import importlib
import logging
import sys
import weakref

log = logging.getLogger(__name__)

# Kept outside the instances, so that a model pickled into dataloader workers carries no fused state.
_STATE = weakref.WeakKeyDictionary()      # model -> (weights key, fused model), or (None, None) once refused
_DECODER = weakref.WeakKeyDictionary()    # PointPillars bbox_head -> the fused model of the last eval forward


def _builders():
    """Reference class name -> the builder of its fused model (``fused_from_reference`` of its model module)."""
    from . import kpconv, pointpillars, pvcnn, randlanet, sparseconvunet
    return dict(RandLANet=randlanet.fused_from_reference, PointPillars=pointpillars.fused_from_reference,
                KPFCNN=kpconv.fused_from_reference, PVCNN=pvcnn.fused_from_reference,
                SparseConvUnet=sparseconvunet.fused_from_reference)


def patch(model, build):
    """Makes the reference instance `model` run its forward on ``build(model)``, a fused model of the weights it holds
    now, and, when that model decodes boxes (PointPillars), its ``bbox_head.get_bboxes`` too.  The forward raises in
    train mode.  A `build` that raises leaves `model` as it was.  Returns `model`."""
    fused = build(model)

    def forward(inputs):
        if model.training:
            raise RuntimeError("open3d_ml_b200: the fused %s path is inference-only" % type(model).__name__)
        return fused.forward(inputs)
    model.forward = forward
    if hasattr(fused, "get_bboxes"):
        model.bbox_head.get_bboxes = fused.get_bboxes
    return model


def _weights_key(model):
    # in-place writes (load_state_dict, optimiser steps, BN statistics) bump _version; .to() moves the storage
    return [(t.data_ptr(), t._version) for ts in (model.parameters(), model.buffers()) for t in ts]


def _fused(model, build):
    """The fused model of the weights `model` holds now, or None when the fused path refuses its config."""
    key = _weights_key(model)
    state = _STATE.get(model)
    if state is not None and (state[1] is None or state[0] == key):
        return state[1]
    name = type(model).__name__
    try:
        fused = build(model)
    except RuntimeError as e:
        log.warning("open3d_ml_b200: %s runs its reference forward, the fused path refuses its config: %s", name, e)
        _STATE[model] = (None, None)
        return None
    if state is None:
        log.info("open3d_ml_b200: %s runs its fused forward", name)
    else:
        log.debug("open3d_ml_b200: %s weights changed, fused forward rebuilt", name)
    _STATE[model] = (key, fused)
    return fused


def _wrapped(reference, dispatch):
    dispatch.__wrapped__ = reference
    dispatch.__doc__ = reference.__doc__
    dispatch._o3dml_b200_fused = True
    return dispatch


def _forward(cls, build):
    reference = cls.forward

    def forward(self, *args, **kwargs):
        fused = None if self.training else _fused(self, build)
        head = getattr(self, "bbox_head", None)
        if head is not None:
            # PointPillars: inference_end decodes the maps of this forward through bbox_head.get_bboxes
            _DECODER[head] = fused
        if fused is None:
            return reference(self, *args, **kwargs)
        return fused.forward(*args, **kwargs)
    return _wrapped(reference, forward)


def _get_bboxes(cls):
    reference = cls.get_bboxes

    def get_bboxes(self, *args, **kwargs):
        fused = None if self.training else _DECODER.get(self)
        if fused is None:
            return reference(self, *args, **kwargs)
        return fused.get_bboxes(*args, **kwargs)
    return _wrapped(reference, get_bboxes)


def is_fused(cls):
    """True when ``fuse_reference_models`` has wrapped the forward of the reference class ``cls``."""
    return getattr(cls.forward, "_o3dml_b200_fused", False)


def reference_classes():
    """The reference classes that ``fuse_reference_models`` wraps, by name."""
    import open3d.ml.torch as ml3d
    return {name: getattr(ml3d.models, name) for name in _builders()}


def fuse_reference_models():
    """Wraps the forward of the five reference classes of ``open3d.ml.torch.models`` (see the module doc).
    Idempotent.  Needs ``shim.install`` with a reference root first."""
    if "open3d" not in sys.modules:
        raise RuntimeError("open3d_ml_b200.fuse: call shim.install(ml3d_root) first")
    classes = reference_classes()
    for name, build in _builders().items():
        cls = classes[name]
        if not is_fused(cls):
            cls.forward = _forward(cls, build)
    head = importlib.import_module(classes["PointPillars"].__module__).Anchor3DHead
    if not getattr(head.get_bboxes, "_o3dml_b200_fused", False):
        head.get_bboxes = _get_bboxes(head)
