"""Population play without a GPU: the four entry points are declared and exported and refuse malformed calls at n = 0
(nothing is launched), the pair thresholds match a numpy restatement, and SelfPlayRollout refuses malformed pairs,
pair_weights and combinations before it touches the device."""
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.greedy import GreedyHumanModel
from overcooked_ai_b200.selfplay import (BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout, member_thresholds,
                                         pair_thresholds)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced
SYMS = ("ovc_assign_pairs", "ovc_group_pairs", "ovc_encode_linear_grouped_masked", "ovc_policy_tail_grouped_joint")


def test_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    lib = _native.lib()
    for sym in SYMS:
        assert re.search(r"\b%s\s*\(" % sym, hdr) and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym


def _refused(rc, lib, what):
    return rc != 0 and what in lib.ovc_last_error()


def test_assign_pairs_refuses_malformed_calls():
    lib = _native.lib()
    call = lambda done=A, thr=A, k=3, counter=A, pair=A, rec=A, count=A, cap=2: lib.ovc_assign_pairs(done, thr, k, 0, 0, counter, pair,
                                                                                                     rec, count, cap, None)
    assert call() == 0, lib.ovc_last_error()
    assert call(k=1) == 0 and call(k=64) == 0 and call(done=0, thr=0, counter=0, rec=0, count=0) == 0
    for kw in (dict(pair=0), dict(counter=0), dict(count=0)):
        assert _refused(call(**kw), lib, b"null"), kw
    for kw in ("done", "count"):
        assert _refused(call(**{kw: A + 2}), lib, b"4-byte"), kw
    for kw in ("pair", "rec", "thr", "counter"):
        assert _refused(call(**{kw: A + 4}), lib, b"8-byte"), kw
    for k in (0, 65):
        assert _refused(call(k=k), lib, b"n_members"), k
    assert _refused(call(cap=-1), lib, b"capacity")
    assert _refused(lib.ovc_assign_pairs(A, A, 3, -1, 0, A, A, A, A, 2, None), lib, b"env count")


def test_group_pairs_refuses_malformed_calls():
    lib = _native.lib()
    call = lambda pair=A, k=3, n=0, lst=A, first=A, jrow=A, eo=A, ro=A: lib.ovc_group_pairs(pair, k, n, lst, first, jrow, eo, ro, None)
    assert call() == 0, lib.ovc_last_error()
    assert call(k=1) == 0 and call(k=64) == 0
    for kw in ("pair", "lst", "first", "jrow", "eo", "ro"):
        assert _refused(call(**{kw: 0}), lib, b"null"), kw
    assert _refused(call(pair=A + 4), lib, b"8-byte")
    for kw in ("lst", "first", "jrow", "eo", "ro"):
        assert _refused(call(**{kw: A + 2}), lib, b"4-byte"), kw
    for k in (0, 65):
        assert _refused(call(k=k), lib, b"n_members"), k
    for n in (-1, 2**29):
        assert _refused(call(n=n), lib, b"n_envs"), n


def test_grouped_masked_encode_refuses_malformed_calls():
    lib = _native.lib()
    call = lambda lst=A, first=A, wt=A, off=A, k=3, out=A, n_out=512, n_layouts=1: lib.ovc_encode_linear_grouped_masked(
        A, n_layouts, A, lst, first, wt, A, off, k, out, 0, 16, 5, 4, 400, n_out, 0.2, None)
    assert call() == 0, lib.ovc_last_error()
    assert call(k=1) == 0 and call(k=64) == 0
    for kw in ("lst", "first", "wt", "off", "out"):
        assert _refused(call(**{kw: 0}), lib, b"null"), kw
    for kw in ("lst", "first", "off"):
        assert _refused(call(**{kw: A + 2}), lib, b"aligned"), kw
    assert _refused(call(out=A + 8), lib, b"16-byte")
    for k in (0, 65):
        assert _refused(call(k=k), lib, b"n_members"), k
    assert _refused(call(n_out=96), lib, b"n_out")
    assert _refused(call(n_layouts=9), lib, b"8 layouts")


def test_grouped_joint_tail_refuses_malformed_calls():
    lib = _native.lib()

    def call(n_rows=0, k0=160, k=3, x=A, w=A, bias=A, counter=A, jrow=A, offsets=A, actions=A, values=A, scores=A, logp=A):
        return lib.ovc_policy_tail_grouped_joint(x, n_rows, k0, 0.2, w, bias, w, bias, 2, w, bias, 0.3, 6, 0, counter, jrow, offsets, k,
                                                 actions, values, scores, logp, None)
    assert call() == 0, lib.ovc_last_error()
    assert call(k=1) == 0 and call(k=64) == 0 and call(values=0, scores=0) == 0
    for kw in ("x", "w", "bias", "counter", "jrow", "offsets", "actions", "logp"):
        assert _refused(call(**{kw: 0}), lib, b"null"), kw
    for kw in ("x", "w"):
        assert _refused(call(**{kw: A + 8}), lib, b"16-byte"), kw
    for kw in ("bias", "scores", "counter"):
        assert _refused(call(**{kw: A + 4}), lib, b"8-byte"), kw
    for kw in ("offsets", "actions", "values", "logp", "jrow"):
        assert _refused(call(**{kw: A + 2}), lib, b"4-byte"), kw
    for k in (0, 65):
        assert _refused(call(k=k), lib, b"n_members"), k
    assert _refused(call(k0=48), lib, b"k0")
    assert _refused(call(n_rows=2**31), lib, b"n_rows")


@pytest.mark.parametrize("K", [1, 2, 5, 64])
def test_pair_thresholds_match_a_numpy_restatement(K):
    rng = np.random.RandomState(K)
    w = rng.rand(K, K) * (rng.rand(K, K) > 0.3)
    w[0, 0] += 0.1  # a positive sum
    flat = w.ravel()
    cdf = np.cumsum(flat) / flat.sum()
    want = np.floor(cdf[:-1] * 2.0**32).astype(np.int64)
    assert np.array_equal(pair_thresholds(w, K), want)
    if K * K <= 64:
        assert np.array_equal(pair_thresholds(w, K), member_thresholds(flat))
    # a pair of weight 0 has an empty interval: its threshold equals the one before
    thr = np.concatenate([[0], pair_thresholds(w, K), [2**32]])
    assert all(thr[q + 1] == thr[q] for q in range(K * K) if flat[q] == 0)


def test_pair_thresholds_refuse_malformed_weights():
    with pytest.raises(AssertionError, match="3 x 3"):
        pair_thresholds(np.ones((3, 2)), 3)
    with pytest.raises(AssertionError, match="3 x 3"):
        pair_thresholds(np.ones(9), 3)
    with pytest.raises(AssertionError, match="non-negative"):
        pair_thresholds([[1, -1], [1, 1]], 2)
    with pytest.raises(AssertionError, match="positive sum"):
        pair_thresholds(np.zeros((2, 2)), 2)


def _env(n=8, n_layouts=1, w=5, h=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=w, height=h)] * n_layouts, device=torch.device("cpu"), n_layouts=n_layouts,
                           n_envs=n)


def test_selfplay_refuses_malformed_pairs():
    env, two = _env(8), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)]
    ok = torch.zeros((8, 2), dtype=torch.int32)
    for bad in (torch.zeros((8, 2), dtype=torch.int64), torch.zeros((7, 2), dtype=torch.int32), torch.zeros((8, 3), dtype=torch.int32),
                torch.zeros((2, 8), dtype=torch.int32).t(), ok.numpy()):
        with pytest.raises(AssertionError, match="int32 tensor \\[N, 2\\]"):
            SelfPlayRollout(env, two, pairs=bad)
    for bad in (ok + 2, ok - 1):
        with pytest.raises(AssertionError, match="must lie in \\[0, 2\\)"):
            SelfPlayRollout(env, two, pairs=bad)
    with pytest.raises(AssertionError, match="environments' device"):
        SelfPlayRollout(env, two, pairs=torch.zeros((8, 2), dtype=torch.int32, device="meta"))


def test_selfplay_refuses_malformed_pair_weights():
    env, two = _env(8), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)]
    for bad in ([1.0, 1.0], [[1.0, 1.0, 1.0]] * 2, np.ones((3, 3))):
        with pytest.raises(AssertionError, match="2 x 2"):
            SelfPlayRollout(env, two, pair_weights=bad)
    with pytest.raises(AssertionError, match="non-negative"):
        SelfPlayRollout(env, two, pair_weights=[[1.0, -0.5], [1.0, 1.0]])
    with pytest.raises(AssertionError, match="positive sum"):
        SelfPlayRollout(env, two, pair_weights=[[0.0, 0.0], [0.0, 0.0]])


def test_selfplay_refuses_population_play_with_what_it_excludes():
    env, two = _env(8), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)]
    pairs, uniform = torch.zeros((8, 2), dtype=torch.int32), [[1.0, 1.0], [1.0, 1.0]]
    with pytest.raises(AssertionError, match="pass one of them"):
        SelfPlayRollout(env, two, pairs=pairs, pair_weights=uniform)
    with pytest.raises(AssertionError, match="no blocks"):
        SelfPlayRollout(env, two, pair_weights=uniform, blocks=[4, 4])
    with pytest.raises(AssertionError, match="no partner"):
        SelfPlayRollout(env, two, pairs=pairs, partner=BCPolicy(), bc_factor=0.5)
    with pytest.raises(AssertionError, match="no partner"):
        SelfPlayRollout(env, two, pair_weights=uniform, partner=GreedyHumanModel(), bc_factor=0.5)
    with pytest.raises(AssertionError, match="LSTM member"):
        SelfPlayRollout(env, [RllibShapedCNN(5, 4), RllibLSTMShapedCNN(5, 4)], pair_weights=uniform)
    with pytest.raises(AssertionError, match="autocast_dtype=None"):
        SelfPlayRollout(env, two, pair_weights=uniform, autocast_dtype=None)
    with pytest.raises(AssertionError, match="list model"):
        SelfPlayRollout(env, RllibShapedCNN(5, 4), pair_weights=[[1.0]])


def test_selfplay_refuses_population_play_beyond_k7():
    uniform = [[1.0, 1.0], [1.0, 1.0]]
    with pytest.raises(AssertionError, match="needs K7.*9 layouts"):
        SelfPlayRollout(_env(8, n_layouts=9), [RllibShapedCNN(5, 4)] * 2, pair_weights=uniform)
    with pytest.raises(AssertionError, match="needs K7.*16x16 grid"):  # the 19-plane table of a 16x16 grid exceeds shared memory
        SelfPlayRollout(_env(8, w=16, h=16), [RllibShapedCNN(16, 16)] * 2, pair_weights=uniform)
