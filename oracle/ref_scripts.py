"""oracle/ref_scripts.py -- TEST INFRASTRUCTURE.

Adds to the snapshot of make_ref_snapshot.py (oracle/_ref/, git-ignored) what the unmodified
``scripts/run_pipeline.py`` needs beyond ``ml3d/**/*.py`` and the configs: the script itself, the
``scripts/README.md`` it reads, and the datasets' ``.yaml`` / ``.txt`` resource files (SemanticKITTI's label map,
ScanNet's scene lists), so that the ``-m gpu`` run_pipeline tests can run the script where only the snapshot exists.
Run by __graft_entry__.build() after make_ref_snapshot.snapshot().  Nothing here is imported by the product package.
"""
import os
import shutil

from oracle.make_ref_snapshot import DST, SRC, live_root

FILES = ("scripts/run_pipeline.py", "scripts/README.md")
RESOURCES = os.path.join("ml3d", "datasets", "_resources")


def copy():
    """Copies FILES and the resource files from the live reference tree into DST.  -> the number of files, or None
    where there is no live tree."""
    if live_root() is None:
        return None
    rels = list(FILES)
    for root, _, files in os.walk(os.path.join(SRC, RESOURCES)):
        rels += [os.path.relpath(os.path.join(root, f), SRC) for f in files if f.endswith((".yaml", ".txt"))]
    for rel in rels:
        out = os.path.join(DST, rel)
        os.makedirs(os.path.dirname(out), exist_ok=True)
        shutil.copyfile(os.path.join(SRC, rel), out)
    return len(rels)


if __name__ == "__main__":
    print(copy())
