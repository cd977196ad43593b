#!/usr/bin/env python
"""Import the reference's layout DATA files into overcooked_ai_b200/data/layouts.json.

The reference stores each layout as a Python dict literal in
src/overcooked_ai_py/data/layouts/<name>.layout (loader: utils.py:31-33, 223-226).  Layouts are an
input FORMAT of the hot path (SURVEY.md §2 row 11), and the package must not depend on a checkout of
the reference, so the grids + recipe parameters are normalised once into one JSON document that travels
with the package.  With a checkout of the reference:  OVC_REFERENCE=<checkout> python tools/import_layouts.py
"""
import ast
import glob
import json
import os
import sys

REF = os.environ["OVC_REFERENCE"]
SRC = os.path.join(REF, "src/overcooked_ai_py/data/layouts")
DST = os.path.join(os.path.dirname(__file__), "..", "overcooked_ai_b200", "data", "layouts.json")


def main():
    out = {}
    for path in sorted(glob.glob(os.path.join(SRC, "*.layout"))):
        name = os.path.basename(path)[: -len(".layout")]
        with open(path) as f:
            # tutorial_3 spells its bonus float('inf'); 1e999 is the same value as a literal
            d = ast.literal_eval(f.read().replace("float('inf')", "1e999"))
        d["grid"] = [row.strip() for row in d["grid"].split("\n")]
        out[name] = d
    with open(DST, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote %d layouts to %s" % (len(out), os.path.normpath(DST)))


if __name__ == "__main__":
    sys.exit(main())
