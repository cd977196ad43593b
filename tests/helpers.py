"""Shared fixtures loading for the parity tests."""
import glob
import json
import os

import numpy as np

from overcooked_ai_b200 import layout as L

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EVENT_MASK = (1 << 25) - 1

TRACE_FILES = sorted(glob.glob(os.path.join(GOLD, "trace_*.npz")))
TRACE_IDS = [os.path.basename(p)[len("trace_"):-len(".npz")] for p in TRACE_FILES]


class Trace(object):
    """One golden file: reference transitions for one layout, [E episodes, T steps]."""

    def __init__(self, path):
        d = np.load(path)
        self.name = os.path.basename(path)
        self.params = json.loads(str(d["params"])) if "params" in d else {}
        self.layout_name = str(d["layout"])
        self.layout = L.compile_layout(self.layout_name, **self.params)
        self.tables, self.starts, self.S = L.build_tables([self.layout])
        st, ac = d["states"], d["actions"]
        self.sparse2, self.shaped, self.events = d["sparse"], d["shaped"], d["events"]
        if st.ndim == 2:  # single episode files
            st, ac = st[None], ac[None]
            self.sparse2, self.shaped, self.events = self.sparse2[None], self.shaped[None], self.events[None]
        self.states, self.actions = st, ac
        self.E, self.T = ac.shape[:2]
        self.sparse = self.sparse2.sum(-1)
        self.data = d

    def flat(self):
        """All (state, action, next_state, ...) transitions as one batch."""
        S = self.S
        s0 = np.ascontiguousarray(self.states[:, :-1].reshape(-1, S))
        s1 = self.states[:, 1:].reshape(-1, S)
        a = np.ascontiguousarray(self.actions.reshape(-1, 2))
        return s0, a, s1, self.sparse.reshape(-1), self.shaped.reshape(-1, 2), self.events.reshape(-1, 2)


def lut_bytes(layouts):
    return np.stack([l.feature_lut() for l in layouts]).view(np.uint8).reshape(len(layouts), -1)


def strip_signature(name):
    """A demangled kernel name without return type and parameter list: ``void ovc::k<(int)1>(args)`` /
    ``ovc::k(args)`` -> ``ovc::k<(int)1>`` / ``ovc::k`` (up to the first parenthesis outside the template arguments)."""
    name = name[5:] if name.startswith("void ") else name
    depth = 0
    for i, c in enumerate(name):
        depth += (c == "<") - (c == ">")
        if c == "(" and depth == 0:
            return name[:i]
    return name
