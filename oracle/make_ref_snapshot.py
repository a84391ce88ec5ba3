"""oracle/make_ref_snapshot.py -- TEST INFRASTRUCTURE.

Copies the UNMODIFIED Python reference tree (ml3d/**/*.py, ml3d/configs/*.yml, tests/test_models.py)
from /root/reference into oracle/_ref/ so that the `-m gpu` boundary tests can drive the reference's own
classes, pipelines and smoke tests through open3d_ml_b200.shim on the GPU box, where /root/reference
does not exist.  oracle/_ref/ is git-ignored (never part of the history, like any oracle/_ref artefact)
but not gpurun-ignored, so it travels with the snapshot.  Run by __graft_entry__.build() whenever
/root/reference is present.  Nothing under oracle/_ref is imported by the product package.
"""
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get("OPEN3D_ML_ROOT", "/root/reference")
DST = os.path.join(HERE, "_ref")


def live_root():
    """The unmodified reference tree itself ($OPEN3D_ML_ROOT or /root/reference), or None where it is absent."""
    return SRC if os.path.isdir(os.path.join(SRC, "ml3d")) else None


def snapshot(force=False):
    if live_root() is None:
        return None
    stamp = os.path.join(DST, ".stamp")
    if os.path.exists(stamp) and not force:
        return DST
    n = 0
    for sub, exts in (("ml3d", (".py", ".yml")), ("tests", (".py",))):
        for root, _, files in os.walk(os.path.join(SRC, sub)):
            if "/tf" in root.replace(SRC, "") and sub == "ml3d":
                continue                       # the TensorFlow twin is never imported here
            for f in files:
                if f.endswith(exts):
                    rel = os.path.relpath(os.path.join(root, f), SRC)
                    out = os.path.join(DST, rel)
                    os.makedirs(os.path.dirname(out), exist_ok=True)
                    shutil.copyfile(os.path.join(root, f), out)
                    n += 1
    open(stamp, "w").write("%d files copied from %s\n" % (n, SRC))
    return DST


def ref_root():
    """Where the unmodified reference tree can be imported from: the live tree here, the snapshot on the GPU box."""
    return live_root() or (DST if os.path.isdir(os.path.join(DST, "ml3d")) else None)


if __name__ == "__main__":
    print(snapshot(force="--force" in sys.argv))
