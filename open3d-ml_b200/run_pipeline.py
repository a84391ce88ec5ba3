"""Runs Open3D-ML's unmodified ``scripts/run_pipeline.py`` on this library, with the fused forwards:

    python -m open3d_ml_b200.run_pipeline [--ml3d-root PATH] <run_pipeline.py arguments>

e.g. ``python -m open3d_ml_b200.run_pipeline torch -c ml3d/configs/pvcnn_s3dis.yml --split test --ckpt_path ...``.
The Open3D-ML tree is ``--ml3d-root`` or ``$OPEN3D_ML_ROOT``.  The launcher installs the shim
(``shim.install``) and the fused dispatch (``fuse.fuse_reference_models``), then runs the script as ``__main__`` with
the remaining arguments.  It refuses, before the script runs, the TensorFlow framework and more than one
``--device_ids`` (the script's ``mp.spawn`` path for distributed training, whose workers would not get the shim).
"""
import contextlib
import importlib
import io
import os
import runpy
import sys


def _split(argv):
    """-> (the --ml3d-root value or None, the script's arguments)."""
    root, rest, i = None, [], 0
    while i < len(argv):
        a = argv[i]
        if a == "--ml3d-root":
            if i + 1 == len(argv):
                raise SystemExit("open3d_ml_b200.run_pipeline: --ml3d-root needs a path")
            root, i = argv[i + 1], i + 2
            continue
        if a.startswith("--ml3d-root="):
            root = a.split("=", 1)[1]
        else:
            rest.append(a)
        i += 1
    return root, rest


def _script_args(script, argv):
    """The script's own parse_args() on `argv`, quietly (the script prints its arguments again when it runs)."""
    ns = runpy.run_path(script, run_name="open3d_ml_b200_run_pipeline_args")
    saved, sys.argv = sys.argv, [script] + argv
    out = io.StringIO()
    try:
        with contextlib.redirect_stdout(out):
            return ns["parse_args"]()[0]
    except SystemExit:
        sys.stdout.write(out.getvalue())      # --help, or the parser's own usage error
        raise
    finally:
        sys.argv = saved


def install(root):
    """The shim for `root`, and the registries the script looks its pipeline, model and dataset up in."""
    from . import shim
    shim.install(root)
    # Open3D's open3d.ml.torch imports ml3d.torch, whose import registers the pipelines, models and datasets that
    # the script looks up by name; the shim resolves its submodules lazily
    importlib.import_module("ml3d.torch")
    importlib.import_module("ml3d.datasets")


def prepare(argv):
    """Checks the launch and installs the shim.  -> (script path, script arguments).  Raises SystemExit with a
    message for a launch that cannot run here."""
    root, rest = _split(argv)
    root = root or os.environ.get("OPEN3D_ML_ROOT")
    if not root:
        raise SystemExit("open3d_ml_b200.run_pipeline: no Open3D-ML tree: pass --ml3d-root PATH or set OPEN3D_ML_ROOT")
    root = os.path.abspath(root)
    script = os.path.join(root, "scripts", "run_pipeline.py")
    if not os.path.isdir(os.path.join(root, "ml3d")) or not os.path.isfile(script):
        raise SystemExit("open3d_ml_b200.run_pipeline: %s is not an Open3D-ML tree (it needs ml3d/ and "
                         "scripts/run_pipeline.py)" % root)
    install(root)
    args = _script_args(script, rest)
    from open3d.ml.utils import convert_device_name, convert_framework_name
    if convert_framework_name(args.framework) != "torch":
        raise SystemExit("open3d_ml_b200.run_pipeline: framework '%s': this library runs the torch models only"
                         % args.framework)
    device, ids = convert_device_name(args.device, args.device_ids)
    if device != "cpu" and len(ids) > 1:
        raise SystemExit("open3d_ml_b200.run_pipeline: --device_ids %s: distributed runs (mp.spawn) are not supported"
                         "; pass one device id" % " ".join(map(str, args.device_ids)))
    return script, rest


def main(argv=None):
    script, rest = prepare(sys.argv[1:] if argv is None else list(argv))
    from .fuse import fuse_reference_models
    fuse_reference_models()
    sys.argv = [script] + rest
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
