"""Every compiled form of the environment kernels against the CPU oracle.

``INSTANTIATIONS`` names each device entry point of the library that is not a policy kernel, as ``cuobjdump -symbols |
cu++filt`` prints it without its parameter list (tests/test_env_forms_cpu.py checks that this table and the policy table
of tests/test_gpu_policy_forms.py together are exactly what the built library holds), and says which test compares it
with the oracle: a case of this file, or another test that already does.

K1 (``step_kernel``: one transition, and the multi-step path that rollouts fall back to for record I/O 2 / 3 and for
more than 8 layouts) and K5 (``rollout_kernel``) have a case per instantiation: S from ``state_words`` or a 128-word
layout, RS from random start states, IO from the environment's record I/O, WIDE / FMT from the action and output formats,
the tile from the number of layouts (3 or more: 128 environments at S <= 32) or from ``OVC_K5_TILE=32`` in a child
process.  Each case runs consecutive launches of a random interact-biased trace on environment counts that are neither a
multiple of 32 nor of the tile, with episodes cut by the horizon inside launches, and compares the rewards, events and
dones of every transition and the records after every launch with the oracle bit for bit.  It also proves which form it
ran: the kernels ``torch.profiler`` saw must include the table key.

K5 skips its L2 action prefetch in one-wave grids outside 12-24 warps per SM, which is where the small cases run.  Each
K5 form therefore has a second case on a grid of more than 32 CTAs per SM (sm_90's limit on resident CTAs, so more than
one wave whatever the occupancy), where the prefetch is on, and there the oracle replays every environment."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import limit_layouts as LL
from helpers import strip_signature
from oracle import cpu
from overcooked_ai_b200 import _native, wire
from overcooked_ai_b200.batched import BatchedOvercookedEnv

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FMTS = {"wide": 0, "host": 1, "stream": 2}
IO_NAME = {1: _native.IO_TMA_TENSOR, 2: _native.IO_TMA_BULK, 3: _native.IO_DIRECT}


def _instantiations():
    t = {}
    for S in (16, 32, 64, 128):
        for rs in (0, 1):
            for io in (1, 2, 3):
                for wide in (0, 1):
                    t["ovc::step_kernel<(int)%d, (int)%d, (bool)%d, (bool)%d>" % (S, io, rs, wide)] = ("k1", S, io, rs, wide)
            for tile in ((32, 64, 128) if S <= 32 else (64,)):
                for fmt in FMTS:
                    t["ovc::rollout_kernel<(int)%d, (int)%d, (bool)%d, (int)%d>" % (S, tile, rs, FMTS[fmt])] = ("k5", S, tile, rs, fmt)
    parity = "test_gpu_parity.py::"
    for dt in ("float", "__nv_bfloat16", "int", "unsigned char"):
        t["ovc::encode_kernel<%s>" % dt] = "test_gpu_layout_limits.py::test_k2_lossless_encoding_every_dtype"
    t["ovc::reset_kernel"] = parity + "test_reset_mask_and_noop_properties"
    t["ovc::reset_random_kernel"] = parity + "test_random_start_states_vs_oracle_mirror"
    t["ovc::featurize_kernel"] = parity + "test_mixed_layout_observations_vs_oracle"
    t["ovc::potential_kernel"] = parity + "test_potential_kernel_bit_exact_vs_reference"
    for rs in (0, 1):
        t["ovc::potential_shaping_kernel<(bool)%d>" % rs] = "test_gpu_phi_reward.py::test_potential_shaping_vs_oracle"
    for st in (0, 1):
        t["ovc::accumulate_returns_kernel<(bool)%d>" % st] = ("test_gpu_episode_stats.py::test_collect_episodes_vs_oracle_replay" if st
                                                               else parity + "test_accumulate_returns_kernel")
        t["ovc::record_transition_view_kernel<(bool)%d>" % st] = "test_gpu_pair_collect.py::test_record_view_equals_two_view_rows"
        for one_view in (0, 1):
            t["ovc::record_transition_dense_kernel<(bool)%d, (bool)%d>" % (st, one_view)] = "test_gpu_phi_reward.py::test_record_transition_dense_vs_restatement"
    t["ovc::gae_kernel<float>"] = "test_gpu_pair_collect.py::test_gae_view_equals_the_float32_loop_and_the_two_row_kernel"
    t["ovc::gae_kernel<float2>"] = "test_gpu_ppo_collect.py::test_gae_kernel_bit_exact_vs_float32_loop"
    t["ovc::partner_policy_kernel"] = "test_gpu_bc_partner.py::test_k10_exact_on_random_rollouts"
    t["ovc::assign_partners_kernel"] = "test_gpu_bc_partner.py::test_assign_partners_matches_the_restatement"
    t["ovc::learner_rows_kernel"] = "test_gpu_selfplay_mixture.py::test_learner_rows_matches_the_restatement"
    t["ovc::group_members_kernel"] = "test_gpu_population.py::test_group_members_is_a_stable_counting_sort"
    t["ovc::assign_members_kernel"] = "test_gpu_population.py::test_assign_members_matches_the_restatement_and_the_record_slot_rule"
    t["ovc::group_pairs_kernel"] = "test_gpu_population_play.py::test_group_pairs_matches_the_restatement"
    t["ovc::assign_pairs_kernel"] = "test_gpu_population_play.py::test_assign_pairs_matches_the_restatement_and_the_record_slot_rule"
    return t


INSTANTIATIONS = _instantiations()


def _cases(kind):
    return [v[1:] for v in INSTANTIATIONS.values() if isinstance(v, tuple) and v[0] == kind]


def _key(case):
    """The table key of a K1 (S, IO, RS, WIDE) or K5 (S, TILE, RS, FMT) case."""
    if isinstance(case[3], str):
        return "ovc::rollout_kernel<(int)%d, (int)%d, (bool)%d, (int)%d>" % (case[0], case[1], case[2], FMTS[case[3]])
    return "ovc::step_kernel<(int)%d, (int)%d, (bool)%d, (bool)%d>" % case


def _case_id(case):
    return "S%d_%s%d_rs%d_%s" % (case[0], "tile" if isinstance(case[3], str) else "io", case[1], case[2],
                                 case[3] if isinstance(case[3], str) else ("wide" if case[3] else "narrow"))


def canonical(name):
    """A kernel name as the profiler or cu++filt spells it, reduced to ``ns::kernel<a,b,...>``: no return type, no
    parameter list, no ``(int)`` / ``(bool)`` casts, booleans as 0 / 1."""
    name = strip_signature(name.strip())
    name = re.sub(r"\((?:int|bool|unsigned int|ovc::[A-Za-z]+)\)", "", name)
    name = re.sub(r"\btrue\b", "1", re.sub(r"\bfalse\b", "0", name))
    return name.replace(" ", "")


def _launched(fn):
    """Runs fn() under torch.profiler and returns the canonical names of the CUDA kernels it launched."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {canonical(e.name) for e in prof.events() if e.device_type.name == "CUDA"}


# ----------------------------------------------------------------------------------------------------------- cases
def _layouts(S, n_layouts):
    """(layouts, state_words) of S words per record: cramped_room alone fits 16, the classic 9x5 layouts 32; 64 is forced;
    128 is the 124-object-cell 16x16 layout of tests/limit_layouts.py."""
    if S == 16:
        return ["cramped_room"] * n_layouts, None
    if S == 128:
        return ([LL.l16()] + ["cramped_room", "counter_circuit"] * 5)[:n_layouts], None
    names = ["asymmetric_advantages", "counter_circuit", "cramped_room", "coordination_ring", "forced_coordination"] * 2
    return names[:n_layouts], (64 if S == 64 else None)


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


def _launch(env, acts, act_fmt, out_fmt):
    """One call on the trace acts [T, N, 2]: env.step() for a single int32 transition in the int32 format, else one
    rollout in the given formats.  Returns (sparse, shaped, done, events) as host arrays."""
    T = acts.shape[0]
    if T == 1 and act_fmt == "int32" and out_fmt == "int32":
        return [x.cpu().numpy()[None] for x in env.step(torch.from_numpy(acts[0]).cuda())]
    d = _device_actions(np.ascontiguousarray(acts), act_fmt)
    if out_fmt == "int32":
        return [x.cpu().numpy() for x in env.rollout(d)]
    if out_fmt == "narrow":
        return [x.cpu().numpy() for x in env.rollout(d, out=env.alloc_rollout_out(T, narrow=True))]
    if out_fmt == "packed":
        sparse, shaped, _, words = env.rollout(d, out=env.alloc_rollout_out(T, packed=True))
        events, done = wire.decode_event_codes(words.cpu().numpy())
        return [sparse.cpu().numpy(), shaped.cpu().numpy(), done, events]
    if out_fmt == "codes":
        dense = env.expand_codes(env.rollout(d, out=env.alloc_rollout_out(T, codes=True))[3].cpu(), events=True)
    else:  # the sparse event stream, with room for every word
        masks, values, _ = env.rollout_stream(d, cap=min(32 * T, _native.STREAM_CAP_MAX))
        dense, over = env.expand_stream(masks.cpu(), values.cpu().contiguous(), events=True)
        assert over == 0
    return [dense[k].numpy() for k in ("sparse", "shaped", "done", "events")]


# (action format, output format) of the launches that leave the int32 form.  A case takes them launch by launch from its
# own offset, so every such form runs several pairs, and any two consecutive launches include an output format that
# stores the reward values (int32, narrow, packed) besides the code words, which carry no sparse reward.
HOST_FORMATS = [("u8", "int32"), ("packed", "codes"), ("int32", "narrow"), ("u8", "packed"), ("packed", "narrow"), ("int32", "codes")]
ACTION_FORMATS = ["int32", "u8", "packed"]


def _formats(i, j, fmt):
    """(action, output) format of launch j of the case at index i among the cases of its format."""
    if fmt in ("wide", 1):
        return "int32", "int32"
    if fmt == "stream":
        return ACTION_FORMATS[(i + j) % 3], "stream"
    return HOST_FORMATS[(i + j) % len(HOST_FORMATS)]


def run_case(case, big=False):
    """Runs one K1 / K5 case against the oracle and returns the canonical names of the kernels it launched.
    big: a K5 case on a grid of more than 32 CTAs per SM (the prefetch is on), every environment against the oracle.

    What varies from case to case (environment count, launch lengths, layouts, auto-reset, formats) is keyed on the
    case's index among the cases of its kind and format, so that every format sees every variation."""
    k5 = isinstance(case[3], str)
    i = sorted(c for c in _cases("k5" if k5 else "k1") if c[3] == case[3]).index(case)
    S, io, rs = case[0], (1 if k5 else case[1]), case[2]
    if k5:
        n_layouts = 3 if case[1] == 128 else 1 + (i // 2) % 2  # 3 or more layouts: the 128-environment tile at S <= 32
    else:
        # IO 1 runs the multi-step path only with more than 8 layouts (the tables then stay in global memory)
        n_layouts = 9 if io == 1 or (i // 2) % 2 else 2
    if big:
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        n = 32 * n_sm * case[1] + 4321  # > 32 CTAs per SM: more than one wave whatever the occupancy
        launches, horizon = [6, 13], 10
    else:
        n = (517, 1237, 3001)[i % 3]
        launches = ([2, 5, 33], [3, 17, 40])[(i // 2) % 2] if k5 else [1, 1, 6, 1, 30]
        horizon = 25
    auto_reset = big or i % 5 != 2  # some cases keep finished episodes standing (stepped-after-done outputs)
    legs = [(_layouts(S, n_layouts), n, horizon, launches)]
    if not k5 and io == 1:  # and single transitions with the tables in shared memory (at most 8 layouts)
        legs.append((_layouts(S, 2), n, 4, [1] * 6))
    rsd = cpu.random_start(13 + i, 0.5, True) if rs else None
    kw = dict(random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=13 + i) if rs else {}
    runs = []
    for leg, ((layouts, sw), n_leg, hz, lens) in enumerate(legs):
        env = BatchedOvercookedEnv(layouts, n_leg, horizon=hz, auto_reset=auto_reset, state_words=sw, io=IO_NAME[io], **kw)
        assert env.state_words == S and env.n_layouts == len(layouts)
        runs.append((env, hz, lens, _actions(np.random.RandomState(1000 + 7 * i + leg), sum(lens), n_leg)))
    seen = {"done": False, "shaped": False}

    def body():
        for env, hz, lens, acts in runs:
            ref = env.state.cpu().numpy().copy()
            t0 = 0
            for j, length in enumerate(lens):
                t1 = t0 + length
                act_fmt, out_fmt = _formats(i, j, case[3])
                want = cpu.rollout(env._tab_host, env._starts_host, ref, acts[t0:t1], horizon=hz, flags=int(auto_reset), rs=rsd)
                got = _launch(env, acts[t0:t1], act_fmt, out_fmt)
                for k, g, w in zip(("sparse", "shaped", "done", "events"), got, want):
                    assert np.array_equal(g.reshape(w.shape), w), (_case_id(case), act_fmt, out_fmt, length, t0, k)
                assert np.array_equal(env.state.cpu().numpy(), ref), (_case_id(case), act_fmt, out_fmt, length, t0, "record")
                seen["done"] |= bool(want[2].any())
                seen["shaped"] |= bool(want[1].any())
                t0 = t1

    names = _launched(body)
    assert seen["done"] and seen["shaped"], "premise: episodes end inside the trace and shaped rewards are granted"
    return names


# ------------------------------------------------------------------------------------------------------------ K1
K1_CASES = sorted(_cases("k1"))


@pytest.mark.parametrize("case", K1_CASES, ids=_case_id)
def test_k1_form_vs_oracle(case):
    names = run_case(case)
    assert canonical(_key(case)) in names, (_key(case), sorted(names))


# ------------------------------------------------------------------------------------------------------------ K5
K5_CASES = sorted(_cases("k5"))
K5_TILE32 = [c for c in K5_CASES if c[1] == 32]


@pytest.fixture(scope="module")
def tile32_results():
    """The TILE-32 cases, small and big, in one child process with OVC_K5_TILE=32 (read once per process)."""
    code = r"""
import json, sys, traceback
sys.path.insert(0, %r)
import test_gpu_env_forms as F
res = {}
for case in F.K5_TILE32:
    for big in (False, True):
        try:
            res[repr((case, big))] = sorted(F.run_case(case, big=big))
        except Exception:
            res[repr((case, big))] = "FAIL " + traceback.format_exc()[-3000:]
print("RESULTS " + json.dumps(res))
""" % HERE
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800,
                         env=dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]), OVC_K5_TILE="32"))
    lines = [l for l in out.stdout.splitlines() if l.startswith("RESULTS ")]
    assert out.returncode == 0 and lines, out.stdout[-2000:] + out.stderr[-3000:]
    return json.loads(lines[-1][len("RESULTS "):])


def _k5(case, big, tile32_results):
    if case[1] == 32:
        names = tile32_results[repr((case, big))]
        assert not isinstance(names, str), names
        names = set(names)
    else:
        names = run_case(case, big=big)
    assert canonical(_key(case)) in names, (_key(case), sorted(names))


@pytest.mark.parametrize("case", K5_CASES, ids=_case_id)
def test_k5_form_vs_oracle(case, request):
    _k5(case, False, request.getfixturevalue("tile32_results") if case[1] == 32 else None)


@pytest.mark.parametrize("case", K5_CASES, ids=_case_id)
def test_k5_form_with_the_prefetch_vs_oracle(case, request):
    _k5(case, True, request.getfixturevalue("tile32_results") if case[1] == 32 else None)
