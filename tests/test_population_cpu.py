"""A population of partners without a GPU: the new entry points are declared and exported, malformed calls are refused at
n = 0 (nothing is launched), AgentPairRollout refuses a malformed population, and the host's draw table is its float64
definition."""
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, member_thresholds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("ovc_group_members", "ovc_assign_members", "ovc_encode_linear_rows", "ovc_wide_layers_range", "ovc_policy_tail_rows",
           "ovc_sample_actions_rows")
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced


def test_population_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    for sym in SYMBOLS:
        assert sym in declared and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == 5


def _calls(lib, ptr=A, seat=0, k=3, rows=A):
    """Each new entry point with ``ptr`` for a 4-byte-aligned pointer argument, at a size that launches nothing."""
    return {
        "group_members": lambda: lib.ovc_group_members(ptr, k, 0, A, A, None),
        "assign_members": lambda: lib.ovc_assign_members(ptr, A, k, 0, 0, A, A, A, A, 1, None),
        "encode_linear_rows": lambda: lib.ovc_encode_linear_rows(A, 1, A, ptr, seat, rows, A, A, A, A, 0, 16, 5, 4, 400, 512, 0.2, None),
        "wide_layers_range": lambda: lib.ovc_wide_layers_range(A, 0, 512, A, A, 512, A, A, 160, 0.2, rows, ptr, None),
        "policy_tail_rows": lambda: lib.ovc_policy_tail_rows(A, 0, 160, 0.2, A, A, A, A, 2, A, A, 0.3, 6, 0, A, ptr, seat, rows, A, A,
                                                             A, A, A, None),
        "sample_actions_rows": lambda: lib.ovc_sample_actions_rows(A, 8, 6, 0, 0, A, ptr, seat, rows, A, A, A, None),
    }


def test_population_entry_points_accept_well_formed_empty_calls_and_refuse_malformed_ones():
    lib = _native.lib()
    for name, call in _calls(lib).items():
        assert call() == 0, (name, lib.ovc_last_error())
    for name, call in _calls(lib, ptr=A + 2).items():
        assert call() != 0 and b"aligned" in lib.ovc_last_error(), name
    for name, call in _calls(lib, rows=0).items():
        if name not in ("group_members", "assign_members"):
            assert call() != 0 and b"null" in lib.ovc_last_error(), name
    for name, call in _calls(lib, rows=A + 2).items():
        if name not in ("group_members", "assign_members", "wide_layers_range"):  # K9 at m = 0 checks the range pointer's alignment
            assert call() != 0 and b"aligned" in lib.ovc_last_error(), name
    assert lib.ovc_wide_layers_range(A, 0, 512, A, A, 512, A, A, 160, 0.2, A + 2, A, None) != 0
    for name in ("encode_linear_rows", "policy_tail_rows", "sample_actions_rows"):
        for seat in (2, -1):
            assert _calls(lib, seat=seat)[name]() != 0 and b"seat" in lib.ovc_last_error(), (name, seat)
    for name in ("group_members", "assign_members"):
        for k in (0, 65):
            assert _calls(lib, k=k)[name]() != 0 and b"n_members" in lib.ovc_last_error(), (name, k)
        assert _calls(lib, k=64)[name]() == 0
    # null pointers: member / order / offsets; assign_members' member, a draw without a counter, records without count
    assert lib.ovc_group_members(0, 3, 0, A, A, None) != 0 and b"null" in lib.ovc_last_error()
    assert lib.ovc_group_members(A, 3, 0, A, 0, None) != 0
    assert lib.ovc_assign_members(0, A, 3, 0, 0, A, 0, 0, 0, 0, None) != 0 and b"null" in lib.ovc_last_error()
    assert lib.ovc_assign_members(0, A, 3, 0, 0, 0, A, 0, 0, 0, None) != 0 and b"null" in lib.ovc_last_error()
    assert lib.ovc_assign_members(0, 0, 3, 0, 0, 0, A, A, 0, 1, None) != 0 and b"null" in lib.ovc_last_error()
    assert lib.ovc_assign_members(0, 0, 3, 0, 0, 0, A, 0, 0, 0, None) == 0  # a fixed member without records: nothing to do
    assert lib.ovc_assign_members(0, A + 4, 3, 0, 0, A, A, 0, 0, 0, None) != 0 and b"8-byte" in lib.ovc_last_error()
    assert lib.ovc_assign_members(0, 0, 3, 0, 0, 0, A, A, A, -1, None) != 0 and b"capacity" in lib.ovc_last_error()


def _env(n=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n)


def test_agent_pair_refuses_a_malformed_population():
    env, A_, B_ = _env(), RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    with pytest.raises(AssertionError, match="LSTM member"):
        AgentPairRollout(env, (A_, [B_, RllibLSTMShapedCNN(5, 4)]))
    with pytest.raises(AssertionError, match="agent 1 only"):
        AgentPairRollout(env, ([A_, B_], B_))
    with pytest.raises(AssertionError, match="1..64"):
        AgentPairRollout(env, (A_, []))
    with pytest.raises(AssertionError, match="1..64"):
        AgentPairRollout(env, (A_, [BCPolicy()] * 65))
    with pytest.raises(AssertionError, match="pass one of them"):
        AgentPairRollout(env, (A_, [B_, BCPolicy()]), member=torch.zeros(4, dtype=torch.int32), member_weights=[1, 1])
    with pytest.raises(AssertionError, match="go with a population"):
        AgentPairRollout(env, (A_, B_), member_weights=[1.0])
    for w in ([1.0, -1.0], [0.0, 0.0], [1.0, float("nan")]):
        with pytest.raises(AssertionError, match="non-negative"):
            AgentPairRollout(env, (A_, [B_, BCPolicy()]), member_weights=w)
    with pytest.raises(AssertionError, match="one weight per member"):
        AgentPairRollout(env, (A_, [B_, BCPolicy()]), member_weights=[1.0])
    for bad in ([0, 1, 2, 0], [0, -1, 1, 0]):
        with pytest.raises(AssertionError, match=r"\[0, 2\)"):
            AgentPairRollout(env, (A_, [B_, BCPolicy()]), member=torch.tensor(bad, dtype=torch.int32))


def test_member_thresholds_match_their_float64_definition():
    rng = np.random.default_rng(3)
    cases = [[1.0], [1.0, 1.0], [0.0, 1.0, 2.0, 0.0], [0.0, 0.0, 5.0], [3.0, 0.0, 0.0], [1e-300, 1.0], list(rng.random(64)),
             [0.1] * 10, [0.0] * 63 + [1.0]]
    for w in cases:
        thr = member_thresholds(w)
        w64 = np.asarray(w, dtype=np.float64)
        c = np.cumsum(w64)
        assert thr.dtype == np.int64 and thr.shape == (len(w) - 1,)
        for k in range(len(w) - 1):
            assert thr[k] == int(np.floor(c[k] / c[-1] * 2.0**32)), (w, k)
        # the draw member = #{k : w0 >= thr[k]} never gives a zero-weight member, for any 32-bit word
        words = np.concatenate([np.array([0, 1, 2**31, 2**32 - 2, 2**32 - 1], dtype=np.int64), thr, np.maximum(thr - 1, 0)])
        words = words[(words >= 0) & (words < 2**32)]
        drawn = (words[:, None] >= thr[None, :]).sum(1)
        assert np.all(w64[drawn] > 0), (w, drawn)
    assert list(member_thresholds([0.0, 1.0, 2.0, 0.0])) == [0, 2**32 // 3, 2**32]
