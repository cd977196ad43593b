"""The potential-based dense reward (use_phi) without a GPU: the new entry points are declared and exported, malformed
calls are refused at n = 0 (nothing is launched), and the rollouts refuse use_phi on an env without auto_reset."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN, SelfPlayRollout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("ovc_potential_shaping", "ovc_record_transition_dense")
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced
OVC_E_BADARG = -1


def test_phi_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    for sym in SYMBOLS:
        assert sym in declared and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == 5


def _shaping(lib, **kw):
    """ovc_potential_shaping at n = 0 with every argument well formed unless overridden."""
    a = dict(layouts=A, n_layouts=1, start=A, pt=A, cost=A, gpow=A, n_pow=8, state=A, done=A, phi_s=A, dense=A, n=0, S=16)
    a.update(kw)
    return lib.ovc_potential_shaping(a["layouts"], a["n_layouts"], a["start"], a["pt"], a["cost"], a["gpow"], a["n_pow"], a["state"],
                                     a["done"], a["phi_s"], a["dense"], a["n"], a["S"], None, None)


def _dense(lib, **kw):
    """ovc_record_transition_dense at n = 0 with every argument well formed unless overridden."""
    a = dict(sparse=A, shaped=A, dense=A, done=A, factor=A, n=0, one_view=0, rewards=A, dones=A)
    a.update(kw)
    return lib.ovc_record_transition_dense(a["sparse"], a["shaped"], a["dense"], a["done"], a["factor"], a["n"], a["one_view"],
                                           a["rewards"], a["dones"], None, None, None, None)


def _refused(rc, lib, what):
    return rc == OVC_E_BADARG and what in lib.ovc_last_error()


def test_potential_shaping_refuses_malformed_arguments():
    lib = _native.lib()
    assert _shaping(lib) == 0, lib.ovc_last_error()
    for k in ("layouts", "start", "pt", "cost", "gpow", "state", "done", "phi_s", "dense"):
        assert _refused(_shaping(lib, **{k: 0}), lib, b"null"), k
    assert _refused(_shaping(lib, n_pow=1), lib, b"power table")
    for S in (4, 8, 24):
        assert _refused(_shaping(lib, S=S), lib, b"state_words"), S
    assert _refused(_shaping(lib, phi_s=A + 4), lib, b"phi_s must be 8-byte aligned")
    for k in ("dense", "done"):
        assert _refused(_shaping(lib, **{k: A + 2}), lib, b"4-byte aligned"), k
    assert _refused(_shaping(lib, n=-1), lib, b"negative n_envs")


def test_record_transition_dense_refuses_malformed_arguments():
    lib = _native.lib()
    for one_view in (0, 1):
        assert _dense(lib, one_view=one_view) == 0, lib.ovc_last_error()
        assert _dense(lib, one_view=one_view, rewards=0) == 0  # rewards are optional, as in ovc_record_transition
    for k in ("sparse", "shaped", "dense", "factor"):
        assert _refused(_dense(lib, **{k: 0}), lib, b"null"), k
    assert _refused(_dense(lib, done=0), lib, b"null")  # dones are written from done
    assert _refused(_dense(lib, dense=A + 2), lib, b"aligned")
    assert _refused(_dense(lib, rewards=A + 4), lib, b"aligned")  # [N][2] rewards are float2
    assert _dense(lib, one_view=1, rewards=A + 4) == 0
    assert _refused(_dense(lib, one_view=1, rewards=A + 2), lib, b"aligned")
    assert _refused(_dense(lib, one_view=2), lib, b"one_view")
    assert _refused(_dense(lib, n=-1), lib, b"negative")


def _env(auto_reset, n=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n,
                           auto_reset=auto_reset)


def test_use_phi_is_refused_without_auto_reset():
    env, model = _env(auto_reset=False), RllibShapedCNN(5, 4)
    with pytest.raises(AssertionError, match="use_phi needs an auto_reset environment"):
        SelfPlayRollout(env, model, use_phi=True)
    with pytest.raises(AssertionError, match="use_phi needs an auto_reset environment"):
        SelfPlayRollout(env, model, partner=BCPolicy(), bc_factor=0.5, use_phi=True)
    with pytest.raises(AssertionError, match="use_phi needs an auto_reset environment"):
        AgentPairRollout(env, (model, BCPolicy()), use_phi=True)
