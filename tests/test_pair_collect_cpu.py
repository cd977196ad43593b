"""AgentPairRollout.collect() without a GPU: the learner-row entry points are declared and exported, malformed calls are
refused at n = 0 (nothing is launched), and collect() / random_seats refuse what they do not support."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("ovc_record_transition_view", "ovc_gae_view")
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced


def test_learner_row_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    for sym in SYMBOLS:
        assert sym in declared and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == 5


def _record(lib, n=0, sparse=A, swap=A, seat=0, rewards=A, factor=A):
    return lib.ovc_record_transition_view(sparse, A, A, factor, n, swap, seat, rewards, A, A, A, None, None)


def _gae(lib, T=0, n=0, rewards=A, adv=A, targets=A):
    return lib.ovc_gae_view(rewards, A, A, A, T, n, 0.99, 0.95, adv, targets, None)


def test_learner_row_entry_points_accept_empty_calls_and_refuse_malformed_ones():
    lib = _native.lib()
    err = lambda: lib.ovc_last_error()
    assert _record(lib) == 0, err()
    assert _record(lib, swap=0) == 0, err()
    assert _record(lib, seat=1) == 0, err()
    assert _gae(lib) == 0 and _gae(lib, T=5) == 0 and _gae(lib, n=7) == 0, err()
    for kw in ({"sparse": 0}, {"rewards": 0}, {"factor": 0}):
        assert _record(lib, **kw) != 0 and b"null" in err(), kw
    for kw in ({"rewards": 0}, {"adv": 0}, {"targets": 0}):
        assert _gae(lib, **kw) != 0 and b"null" in err(), kw
    for seat in (2, -1):
        assert _record(lib, seat=seat) != 0 and b"seat" in err(), seat
    for kw in ({"swap": A + 2}, {"rewards": A + 2}):
        assert _record(lib, **kw) != 0 and b"aligned" in err(), kw
    for kw in ({"rewards": A + 2}, {"adv": A + 2}, {"targets": A + 2}):
        assert _gae(lib, **kw) != 0 and b"aligned" in err(), kw
    assert _record(lib, n=-1) != 0 and b"negative" in err()
    assert _gae(lib, T=-1) != 0 and _gae(lib, n=-1) != 0


def _env(auto_reset=True, n=3):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n,
                           auto_reset=auto_reset, horizon=400, layout_ids=lambda: torch.zeros(n, dtype=torch.int32))


def test_collect_refuses_a_bc_learner_and_an_environment_without_auto_reset():
    with pytest.raises(AssertionError, match="BCPolicy"):
        AgentPairRollout(_env(), (BCPolicy(), RllibShapedCNN(5, 4)), use_graph=False).collect(4, 0.99, 0.95)
    with pytest.raises(AssertionError, match="auto_reset"):
        AgentPairRollout(_env(auto_reset=False), (RllibShapedCNN(5, 4), BCPolicy()), use_graph=False).collect(4, 0.99, 0.95)


def test_random_seats_refuse_a_swap_tensor():
    with pytest.raises(AssertionError, match="random_seats"):
        AgentPairRollout(_env(), (RllibShapedCNN(5, 4), BCPolicy()), swap=torch.zeros(3, dtype=torch.int32), random_seats=True)
