"""A population of self-play learners without a GPU: the grouped K7 / K9 / K8 entry points are declared and exported, malformed calls
are refused at n = 0 (nothing is launched), and SelfPlayRollout refuses a malformed list model or blocks before it touches
the device."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.greedy import GreedyHumanModel
from overcooked_ai_b200.selfplay import BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced


def test_grouped_tail_is_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    assert "ovc_policy_tail_grouped" in declared and "ovc_policy_tail_grouped" in _native.EXPORTED_SYMBOLS
    assert hasattr(lib, "ovc_policy_tail_grouped")


def _grouped(lib, n_rows=0, k0=160, n_hidden=2, n_actions=6, k=3, x=A, w=A, bias=A, counter=A, offsets=A, actions=A, values=A,
             scores=A, logp=A, slope=0.3):
    return lib.ovc_policy_tail_grouped(x, n_rows, k0, 0.2, w, bias, w, bias, n_hidden, w, bias, slope, n_actions, 0, counter, offsets, k,
                                       actions, values, scores, logp, None)


def test_grouped_tail_accepts_a_well_formed_empty_call_and_refuses_malformed_ones():
    lib = _native.lib()
    assert _grouped(lib) == 0, lib.ovc_last_error()
    assert _grouped(lib, k=1) == 0 and _grouped(lib, k=64) == 0
    assert _grouped(lib, values=0, scores=0, logp=0) == 0  # values, scores and logp are optional
    for kw in ("x", "w", "bias", "counter", "offsets", "actions"):
        assert _grouped(lib, **{kw: 0}) != 0 and b"null" in lib.ovc_last_error(), kw
    for kw in ("x", "w"):
        assert _grouped(lib, **{kw: A + 8}) != 0 and b"16-byte" in lib.ovc_last_error(), kw
    for kw in ("bias", "scores", "counter"):
        assert _grouped(lib, **{kw: A + 4}) != 0 and b"8-byte" in lib.ovc_last_error(), kw
    for kw in ("offsets", "actions", "values", "logp"):
        assert _grouped(lib, **{kw: A + 2}) != 0 and b"4-byte" in lib.ovc_last_error(), kw
    for k in (0, -1, 65):
        assert _grouped(lib, k=k) != 0 and b"n_members" in lib.ovc_last_error(), k
    for k0 in (0, 48, 288):
        assert _grouped(lib, k0=k0) != 0 and b"k0" in lib.ovc_last_error(), k0
    assert _grouped(lib, n_hidden=9) != 0 and b"n_hidden" in lib.ovc_last_error()
    for n_act in (0, 8):
        assert _grouped(lib, n_actions=n_act) != 0 and b"n_actions" in lib.ovc_last_error(), n_act
    assert _grouped(lib, slope=1.5) != 0 and b"slopes" in lib.ovc_last_error()
    for n in (-1, 2**31):
        assert _grouped(lib, n_rows=n) != 0 and b"n_rows" in lib.ovc_last_error(), n


def _env(n=8):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n)


def test_selfplay_refuses_a_malformed_population_of_learners():
    env = _env()
    with pytest.raises(AssertionError, match="1..64 members"):
        SelfPlayRollout(env, [])
    with pytest.raises(AssertionError, match="1..64 members"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4)] * 65)
    with pytest.raises(AssertionError, match="LSTM member"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4), RllibLSTMShapedCNN(5, 4)])
    with pytest.raises(AssertionError, match="RllibShapedCNN"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4), BCPolicy()])
    with pytest.raises(AssertionError, match="one architecture"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4, hidden=32)])
    with pytest.raises(AssertionError, match="one architecture"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4, num_filters=16)])
    with pytest.raises(AssertionError, match="no partner"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4)] * 2, partner=BCPolicy(), bc_factor=0.5)
    with pytest.raises(AssertionError, match="no partner"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4)] * 2, partner=GreedyHumanModel(), bc_factor=0.5)
    with pytest.raises(AssertionError, match="blocks go with"):
        SelfPlayRollout(env, RllibShapedCNN(5, 4), blocks=[4, 4])


def test_selfplay_refuses_malformed_blocks():
    env, two = _env(8), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)]
    for blocks in ([8, 0], [9, -1], [3, 4], [4, 5], [8]):
        with pytest.raises(AssertionError, match="blocks"):
            SelfPlayRollout(env, two, blocks=blocks)
    with pytest.raises(AssertionError, match="one environment per member"):
        SelfPlayRollout(_env(2), [RllibShapedCNN(5, 4)] * 3)


def test_grouped_encode_and_wide_layers_are_declared_and_refuse_malformed_calls():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    lib = _native.lib()
    for sym in ("ovc_encode_linear_grouped", "ovc_wide_layers_grouped"):
        assert re.search(r"\b%s\s*\(" % sym, hdr) and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    enc = lambda wt=A, bias=A, off=A, k=3, out=A, n_out=512: lib.ovc_encode_linear_grouped(A, 1, A, wt, bias, off, k, out, 0, 16, 5, 4,
                                                                                           400, n_out, 0.2, None)
    wide = lambda a0=A, w=A, b=A, off=A, k=3, z=A, k0=512, m=0: lib.ovc_wide_layers_grouped(a0, m, k0, w, b, 512, w, b, 160, 0.2, off, k,
                                                                                            z, None)
    for call in (enc, wide):
        assert call() == 0, lib.ovc_last_error()
        assert call(k=1) == 0 and call(k=64) == 0
        assert call(off=0) != 0 and b"null" in lib.ovc_last_error()
        assert call(off=A + 2) != 0 and b"aligned" in lib.ovc_last_error()
        for k in (0, 65):
            assert call(k=k) != 0 and b"n_members" in lib.ovc_last_error(), k
    assert enc(wt=0) != 0 and b"null" in lib.ovc_last_error()
    assert enc(out=A + 8) != 0 and b"16-byte" in lib.ovc_last_error()
    assert enc(n_out=96) != 0 and b"n_out" in lib.ovc_last_error()
    assert wide(z=0) != 0 and b"null" in lib.ovc_last_error()
    assert wide(a0=A + 8) != 0 and b"16-byte" in lib.ovc_last_error()
    assert wide(b=A + 4) != 0 and b"8-byte" in lib.ovc_last_error()
    assert wide(k0=256) != 0 and b"512" in lib.ovc_last_error()
    assert wide(m=2**31) != 0 and b"2^31" in lib.ovc_last_error()
