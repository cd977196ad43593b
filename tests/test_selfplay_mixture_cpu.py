"""Self-play mixtures without a GPU: the new entry points are declared and exported, malformed calls are refused at n = 0
(nothing is launched), and SelfPlayRollout refuses a malformed partner."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("ovc_learner_rows", "ovc_encode_linear_masked", "ovc_policy_tail_joint")
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced


def test_mixture_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    for sym in SYMBOLS:
        assert sym in declared and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == 5


def _calls(lib, ptr=A, n=0, logp=A):
    """Each new entry point with ``ptr`` for its 4-byte-aligned pointer arguments, at a size that launches nothing."""
    return {
        "learner_rows": lambda: lib.ovc_learner_rows(ptr, n, ptr, ptr, ptr, ptr, None),
        "encode_linear_masked": lambda: lib.ovc_encode_linear_masked(A, 1, A, ptr, ptr, A, A, A, n, 16, 5, 4, 400, 512, 0.2, None),
        "policy_tail_joint": lambda: lib.ovc_policy_tail_joint(A, n, 160, 0.2, A, A, A, A, 2, A, A, 0.3, 6, 0, A, ptr, ptr, ptr, ptr, A,
                                                               logp, None),
    }


def test_mixture_entry_points_accept_well_formed_empty_calls_and_refuse_malformed_ones():
    lib = _native.lib()
    for name, call in _calls(lib).items():
        assert call() == 0, (name, lib.ovc_last_error())
    for name, call in _calls(lib, ptr=A + 2).items():
        assert call() != 0 and b"aligned" in lib.ovc_last_error(), name
    for name, call in _calls(lib, ptr=0).items():
        assert call() != 0 and b"null" in lib.ovc_last_error(), name
    for name, call in _calls(lib, n=-1).items():
        assert call() != 0 and b"n" in lib.ovc_last_error(), name
    assert _calls(lib, logp=0)["policy_tail_joint"]() != 0 and b"null" in lib.ovc_last_error()  # the joint K8 always writes logp
    assert lib.ovc_learner_rows(A, 1 << 29, A, A, A, A, None) != 0 and b"2^29" in lib.ovc_last_error()
    assert lib.ovc_policy_tail_joint(A, 1 << 31, 160, 0.2, A, A, A, A, 2, A, A, 0.3, 6, 0, A, A, A, A, A, A, A, None) != 0
    # K7's own checks hold for the masked form: the weights' alignment, n_out, the layout count
    assert lib.ovc_encode_linear_masked(A, 1, A, A, A, A + 8, A, A, 0, 16, 5, 4, 400, 512, 0.2, None) != 0
    assert lib.ovc_encode_linear_masked(A, 1, A, A, A, A, A, A, 0, 16, 5, 4, 400, 100, 0.2, None) != 0
    assert lib.ovc_encode_linear_masked(A, 9, A, A, A, A, A, A, 0, 16, 5, 4, 400, 512, 0.2, None) != 0


def _env(n=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n)


def test_selfplay_refuses_a_malformed_mixture():
    env, A_, B_ = _env(), RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    with pytest.raises(AssertionError, match="LSTM partner"):
        SelfPlayRollout(env, A_, partner=RllibLSTMShapedCNN(5, 4), bc_factor=0.5)
    with pytest.raises(AssertionError, match="LSTM partner or member"):
        SelfPlayRollout(env, A_, partner=[B_, RllibLSTMShapedCNN(5, 4)], bc_factor=0.5)
    with pytest.raises(AssertionError, match="1..63"):
        SelfPlayRollout(env, A_, partner=[], bc_factor=0.5)
    with pytest.raises(AssertionError, match="1..63"):
        SelfPlayRollout(env, A_, partner=[BCPolicy()] * 64, bc_factor=0.5)
    for kw in (dict(member=torch.zeros(4, dtype=torch.int32)), dict(member_weights=[1.0])):
        for partner in (None, B_, BCPolicy()):
            with pytest.raises(AssertionError, match="go with a population"):
                SelfPlayRollout(env, A_, partner=partner, bc_factor=0.5, **kw)
    with pytest.raises(AssertionError, match="a BCPolicy, an RllibShapedCNN"):
        SelfPlayRollout(env, A_, partner=[B_, "B"], bc_factor=0.5)


def test_selfplay_refuses_malformed_members_and_weights():
    """The population's own checks, reached through SelfPlayRollout before anything runs on a device."""
    env, A_, B_ = _env(), RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    with pytest.raises(AssertionError, match="pass one of them"):
        SelfPlayRollout(env, A_, partner=[B_, BCPolicy()], bc_factor=0.5, member=torch.zeros(4, dtype=torch.int32), member_weights=[1, 1])
    for w in ([1.0, -1.0], [0.0, 0.0], [1.0, float("nan")]):
        with pytest.raises(AssertionError, match="non-negative"):
            SelfPlayRollout(env, A_, partner=[B_, BCPolicy()], bc_factor=0.5, member_weights=w)
    with pytest.raises(AssertionError, match="one weight per member"):
        SelfPlayRollout(env, A_, partner=[B_, BCPolicy()], bc_factor=0.5, member_weights=[1.0])
    for bad in ([0, 1, 2, 0], [0, -1, 1, 0]):
        with pytest.raises(AssertionError, match=r"\[0, 2\)"):
            SelfPlayRollout(env, A_, partner=[B_, BCPolicy()], bc_factor=0.5, member=torch.tensor(bad, dtype=torch.int32))
