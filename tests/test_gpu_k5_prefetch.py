"""The fused rollout kernel K5 prefetches each thread's action OVC_K5_PREFETCH rows ahead into L2 (rows 1 .. D-1 in its
prologue, row s + D in transition s, never a row at or past the launch's last), except in launches whose grid is resident
in one wave at fewer than 12 or at least 24 warps per SM (on an H100: 517 envs run without it, 60 007 envs of
cramped_room + counter_circuit, 938 CTAs of 2 warps = 14 warps per SM in one wave, with it).  A prefetch changes no result, so what these tests can show is that the outputs stay
what the CPU oracle computes, bit for bit, on the paths the prefetch adds: launches around the distance (2 to 90
transitions, the ones shorter than the distance included), environment counts that are neither a multiple of 32 nor of
the CTA tile, every action format and every output format, launches cut by the library, and a launch the host runs
without the prefetch.  Rewards, events and dones of every transition and the record after every launch.  The rows a
prefetch addresses are not observable here."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cpu
from overcooked_ai_b200 import wire
from overcooked_ai_b200.batched import BatchedOvercookedEnv

pytestmark = pytest.mark.gpu

NAMES = ["cramped_room", "counter_circuit"]
HORIZON = 25
# one trace cut into consecutive launches of these lengths: 2, D-1, D, D+1 and 2D+1 for D = 2, 4 (the default) and 16
LAUNCHES = [2, 3, 4, 5, 9, 15, 16, 17, 33, 90]


def _np(t):
    return t.cpu().numpy()


def _actions(rng, T, n, p_interact=0.4):
    a = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32)
    a[rng.rand(T, n, 2) < p_interact] = 5
    return a


def _device_actions(acts, fmt):
    if fmt == "int32":
        return torch.from_numpy(acts).cuda()
    if fmt == "u8":
        return torch.from_numpy(acts.astype(np.uint8)).cuda()
    return torch.from_numpy(wire.pack_actions(acts)).cuda()  # one byte per joint action


def _run(env, d, out_fmt, T):
    """One launch in the given output format; (sparse, shaped, done, events) as host arrays."""
    if out_fmt == "int32":
        return [_np(x) for x in env.rollout(d)]
    if out_fmt == "narrow":
        return [_np(x) for x in env.rollout(d, out=env.alloc_rollout_out(T, narrow=True))]
    if out_fmt == "codes":
        out = env.rollout(d, out=env.alloc_rollout_out(T, codes=True))
        dense = env.expand_codes(out[3].cpu(), events=True)
    else:  # the sparse event stream, with room for every word
        masks, values, _ = env.rollout_stream(d, cap=32 * T)
        dense, over = env.expand_stream(masks.cpu(), values.cpu().contiguous(), events=True)
        assert over == 0
    return [dense[k].numpy() for k in ("sparse", "shaped", "done", "events")]


@pytest.mark.parametrize("out_fmt", ["int32", "narrow", "codes", "stream"])
@pytest.mark.parametrize("act_fmt", ["int32", "u8", "packed"])
@pytest.mark.parametrize("n,random_start", [(517, False), (60007, True)], ids=["n517_no_prefetch", "n60007_random_start"])
def test_k5_launches_around_the_prefetch_distance_vs_oracle(n, random_start, act_fmt, out_fmt):
    T = sum(LAUNCHES)
    acts = _actions(np.random.RandomState(n + 11), T, n)
    kw = dict(random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=13) if random_start else {}
    env = BatchedOvercookedEnv(NAMES, n, horizon=HORIZON, auto_reset=True, **kw)
    rs = cpu.random_start(13, 0.5, True) if random_start else None
    ref = _np(env.state).copy()
    t0 = 0
    for length in LAUNCHES:
        t1 = t0 + length
        want = cpu.rollout(env._tab_host, env._starts_host, ref, acts[t0:t1], horizon=HORIZON, flags=1, n_threads=4, rs=rs)
        got = _run(env, _device_actions(np.ascontiguousarray(acts[t0:t1]), act_fmt), out_fmt, length)
        for k, g, w in zip(("sparse", "shaped", "done", "events"), got, want):
            assert np.array_equal(g, w), (length, t0, k)
        assert np.array_equal(_np(env.state), ref), (length, t0)
        t0 = t1
    assert (want[2] != 0).any() and (want[1] != 0).any(), "premise: episodes end and shaped rewards are granted"


@pytest.mark.parametrize("out_fmt", ["int32", "codes"])
def test_k5_one_full_wave_runs_without_the_prefetch_vs_oracle(out_fmt):
    """cramped_room at 131 072 envs: 2 048 CTAs of 2 warps, resident in one wave at 31 warps per SM on an H100 (132 SMs),
    so the host launches K5 without the prefetch.  Launches of 2, 5 and 33 transitions against the oracle."""
    n = 131072
    acts = _actions(np.random.RandomState(21), 40, n)
    env = BatchedOvercookedEnv(["cramped_room"], n, horizon=HORIZON, auto_reset=True)
    ref = _np(env.state).copy()
    t0 = 0
    for length in (2, 5, 33):
        t1 = t0 + length
        want = cpu.rollout(env._tab_host, env._starts_host, ref, acts[t0:t1], horizon=HORIZON, flags=1, n_threads=8)
        act_fmt = "packed" if out_fmt == "codes" else "int32"
        got = _run(env, _device_actions(np.ascontiguousarray(acts[t0:t1]), act_fmt), out_fmt, length)
        for k, g, w in zip(("sparse", "shaped", "done", "events"), got, want):
            assert np.array_equal(g, w), (length, t0, k)
        assert np.array_equal(_np(env.state), ref), (length, t0)
        t0 = t1


@pytest.mark.parametrize("cap", [3, 5])
def test_k5_prefetch_in_launches_cut_by_the_library(cap):
    """A rollout that ovc_rollout cuts into launches of at most `cap` transitions (library test hook, read once: a child
    process): every launch starts from a shifted action pointer and the last one is short (58 = 19 x 3 + 1 = 11 x 5 + 3),
    with launches both shorter and longer than a prefetch distance of 4.  int32, uint8 and one-byte actions."""
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    code = r"""
import numpy as np, torch
from oracle import cpu
from overcooked_ai_b200 import wire
from overcooked_ai_b200.batched import BatchedOvercookedEnv
names, n, T = ["cramped_room", "counter_circuit"], 60007, 58
rng = np.random.RandomState(8)
acts = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32); acts[rng.rand(T, n, 2) < 0.4] = 5
make = lambda: BatchedOvercookedEnv(names, n, horizon=25, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=4)
env = make()
rs = cpu.random_start(4, 0.5, True)
state = env.state.cpu().numpy().copy()
want = cpu.rollout(env._tab_host, env._starts_host, state, acts, horizon=25, flags=1, n_threads=4, rs=rs)
for g, w in zip(env.rollout(torch.from_numpy(acts).cuda()), want):                  # int32 in, int32 out
    assert np.array_equal(g.cpu().numpy(), w)
assert np.array_equal(env.state.cpu().numpy(), state)
env = make()
out = env.alloc_rollout_out(T, narrow=True)                                         # uint8 actions, narrow outputs
for g, w in zip(env.rollout(torch.from_numpy(acts.astype(np.uint8)).cuda(), out=out), want):
    assert np.array_equal(g.cpu().numpy(), w)
assert np.array_equal(env.state.cpu().numpy(), state)
env = make()
out = env.alloc_rollout_out(T, codes=True)                                          # one-byte actions, code words
env.rollout(torch.from_numpy(wire.pack_actions(acts)).cuda(), out=out)
dense = env.expand_codes(out[3].cpu(), events=True)
for k, w in zip(("sparse", "shaped", "done", "events"), want):
    assert np.array_equal(dense[k].numpy(), w), k
assert np.array_equal(env.state.cpu().numpy(), state)
print("CUT_OK")
"""
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, PYTHONPATH=root, OVC_K5_MAX_LAUNCH_STEPS=str(cap)))
    assert out.returncode == 0 and "CUT_OK" in out.stdout, out.stdout[-1000:] + out.stderr[-3000:]
