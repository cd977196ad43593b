"""Recipe for oracle/_ref/: the UNMODIFIED reference package, copied file by file from the checkout named by
OVC_REFERENCE_SRC so that it travels with the tree (oracle/_ref/ is git-ignored: the reference's sources never enter
this repository's history).

TEST / MEASUREMENT INFRASTRUCTURE.  __graft_entry__.build() runs this; bench.py's `cpu_baseline.reference_python` leg
(oracle/ref_python_bench.py) and the `reference`-marked tests import the copy through oracle/refboot.py.  Only what the step / encode path imports is taken:
the package modules, the layout files and the sprite-sheet JSON the visualizer module reads at import (no test
fixtures, fonts or planner pickles).

    python -m oracle.make_ref [--force]
"""
import os
import shutil
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC_ROOT = os.environ.get("OVC_REFERENCE_SRC")  # a checkout of the reference repository
SRC = os.path.join(_SRC_ROOT, "src", "overcooked_ai_py") if _SRC_ROOT else None
DST = os.path.join(_HERE, "_ref", "src", "overcooked_ai_py")
PARTS = ["__init__.py", "static.py", "utils.py", "mdp", "planning", "agents", "visualization", os.path.join("data", "layouts"),
         os.path.join("data", "planners", "__init__.py"), os.path.join("data", "graphics")]


def make(force=False):
    """Returns the path of the copy, or None when no reference checkout is named and no copy exists."""
    if SRC is None or not os.path.isdir(SRC):
        return DST if os.path.isdir(DST) else None
    stamp = os.path.join(DST, ".copied_from")
    if os.path.exists(stamp) and not force:
        return DST
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    for part in PARTS:
        s, d = os.path.join(SRC, part), os.path.join(DST, part)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        if os.path.isdir(s):
            shutil.copytree(s, d, ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "*_mp.pkl", "*_am.pkl"))
        else:
            shutil.copy2(s, d)
    with open(stamp, "w") as f:
        f.write(SRC + "\n")
    return DST


if __name__ == "__main__":
    print(make(force="--force" in sys.argv))
