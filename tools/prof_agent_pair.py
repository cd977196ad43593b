#!/usr/bin/env python
"""Cost of an agent pair at the config-5 shape (cramped_room, 32 768 envs, run(400)), with CUDA events, written as one JSON
file under --out:

  run(T) of AgentPairRollout((PPO, BC)) against SelfPlayRollout(PPO, partner=BC, bc_factor=1), and of
  AgentPairRollout((PPO_A, PPO_B)) against SelfPlayRollout(PPO_A), alternated in one process, 3 times each;
  per-kernel times, best of 3 over 50 launches: K7 one view (N rows) against two views (2N rows), K9 on N against 2N rows,
  K8 with the one-view draw on N rows against the two-view K8 on 2N rows, K11 one view against two views;
  collect(T) of a learner next to a fixed partner (AgentPairRollout(..., random_seats=True).collect): (PPO, BC) against
  SelfPlayRollout(PPO, partner=BC, bc_factor=1).collect, (PPO, frozen PPO) against self-play collect, and (LSTM PPO, BC),
  alternated in one process, 3 times each;
  per-kernel times of the learner-row record and GAE kernels against their two-row forms (best of 3 over 50 launches);
  the card's name and power limit, read in the same run.

    python tools/prof_agent_pair.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200 import _native  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_agent_pair measures on a CUDA device"


def ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


N, T = args.n, args.steps
torch.manual_seed(0)
ppo_a, ppo_b, bc = RllibShapedCNN(5, 4).cuda(), RllibShapedCNN(5, 4).cuda(), BCPolicy().cuda()
env = lambda: BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
runs = {"pair_ppo_bc": AgentPairRollout(env(), (ppo_a, bc), swap=(torch.arange(N, device="cuda") % 2).to(torch.int32), seed=1),
        "ppo_bc_bc_factor_1": SelfPlayRollout(env(), model=ppo_a, seed=1, partner=bc, bc_factor=1.0),
        "pair_ppo_a_ppo_b": AgentPairRollout(env(), (ppo_a, ppo_b), seed=1),
        "selfplay_ppo_a": SelfPlayRollout(env(), model=ppo_a, seed=1)}
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)", "partner": "BCPolicy 96 -> 64 -> 64 -> 6 (K10)"}
for r in runs.values():
    r.run(3)  # capture + warm every shape
torch.cuda.synchronize()
times = {k: [] for k in runs}
for _ in range(3):
    for k, r in runs.items():
        times[k].append(ms(lambda: r.run(T)))
for k, v in times.items():
    out["run_ms_" + k] = v
    out["run_us_per_transition_" + k] = min(v) * 1e3 / T
out["pair_ppo_bc_over_ppo_bc"] = min(times["pair_ppo_bc"]) / min(times["ppo_bc_bc_factor_1"])
out["pair_ppo_a_ppo_b_over_selfplay"] = min(times["pair_ppo_a_ppo_b"]) / min(times["selfplay_ppo_a"])

# collect(T): a learner next to a fixed partner against the same network's PPO_BC / self-play collect
collects = {"pair_ppo_bc": AgentPairRollout(env(), (ppo_a, bc), seed=1, random_seats=True),
            "ppo_bc_bc_factor_1": runs["ppo_bc_bc_factor_1"],
            "pair_ppo_a_frozen_ppo_b": AgentPairRollout(env(), (ppo_a, ppo_b), seed=1, random_seats=True),
            "selfplay_ppo_a": runs["selfplay_ppo_a"],
            "pair_lstm_bc": AgentPairRollout(env(), (RllibLSTMShapedCNN(5, 4).cuda(), bc), seed=1, random_seats=True)}
for r in collects.values():
    r.collect(T, 0.99, 0.98)  # capture + warm
torch.cuda.synchronize()
ctimes = {k: [] for k in collects}
for _ in range(3):
    for k, r in collects.items():
        ctimes[k].append(ms(lambda: r.collect(T, 0.99, 0.98)))
for k, v in ctimes.items():
    out["collect_ms_" + k] = v
out["collect_pair_ppo_bc_over_ppo_bc"] = min(ctimes["pair_ppo_bc"]) / min(ctimes["ppo_bc_bc_factor_1"])
out["collect_pair_ppo_a_frozen_ppo_b_over_selfplay"] = min(ctimes["pair_ppo_a_frozen_ppo_b"]) / min(ctimes["selfplay_ppo_a"])
bp, bs = collects["pair_ppo_bc"]._batches[(T, False)], collects["selfplay_ppo_a"]._batches[(T, False)]
ce = collects["pair_ppo_bc"].env
one = torch.ones(1, device="cuda")
ret = torch.zeros(N, dtype=torch.int64, device="cuda")
record = {"record_transition_view_stats_us": lambda: ce.record_transition_view(one, 1, None, bp.rewards[0], dones=bp.dones[0], ret_sparse=ret,
                                                                               stats=collects["pair_ppo_bc"].stats, records=bp.episodes),
          "record_transition_stats_us": lambda: ce.record_transition(one, rewards=bs.rewards[0], dones=bp.dones[0], ret_sparse=ret,
                                                                     stats=collects["pair_ppo_bc"].stats, records=bp.episodes),
          "gae_view_us": lambda: ce.gae_view(bp.rewards, bp.values, bp.dones, bp.last_values, 0.99, 0.98, bp.advantages, bp.value_targets),
          "gae_two_rows_us": lambda: ce.gae(bs.rewards, bs.values, bs.dones, bs.last_values, 0.99, 0.98, bs.advantages, bs.value_targets)}
for f in record.values():
    f()
torch.cuda.synchronize()
for k, f in record.items():
    out[k] = min(ms(f, reps=50) for _ in range(3)) * 1e3

# per-kernel: one view (N rows) against two views (2N rows)
sp, agent = runs["selfplay_ppo_a"], runs["pair_ppo_bc"].agents[0]
e = sp.env
lib, s = _native.lib(), e._stream()
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
acts = torch.zeros((N, 2), dtype=torch.int32, device="cuda")


def k9(a0, z):
    w1, b1, w2, b2 = sp._wide
    _native.check(lib.ovc_wide_layers(a0.data_ptr(), a0.shape[0], a0.shape[1], w1.data_ptr(), b1.data_ptr(), w1.shape[0], w2.data_ptr(),
                                      b2.data_ptr(), w2.shape[0], 0.2, z.data_ptr(), s))


def k8(z, view):
    w1, b1, wh, bh, wo, bo = sp._tail
    a = (z.data_ptr(), z.shape[0], z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0], wo.data_ptr(),
         bo.data_ptr(), 0.3, 6, 1, counter.data_ptr())
    if view:
        _native.check(lib.ovc_policy_tail_view(*a, 0, 0, acts.data_ptr(), 0, 0, 0, s))
    else:
        _native.check(lib.ovc_policy_tail(*a, acts.data_ptr(), 0, 0, s))


lstm = SelfPlayRollout(e, model=RllibLSTMShapedCNN(5, 4).cuda(), seed=1, use_graph=False)
w, b, wo, bo = lstm._lstm_tables
x2, h2, c2 = lstm._x, lstm.h, lstm.c
x1, h1, c1 = x2[:N].contiguous(), h2[:N].contiguous(), c2[:N].contiguous()


def k11(x, h, c, view):
    head = (x.data_ptr(), h.data_ptr(), c.data_ptr(), e.done.data_ptr(), x.shape[0], w.data_ptr(), b.data_ptr(), wo.data_ptr(),
            bo.data_ptr(), 6, 1, counter.data_ptr())
    tail = (h.data_ptr(), c.data_ptr(), 0, 0, acts.data_ptr(), 0, 0, 0, s)
    _native.check(lib.ovc_lstm_head_view(*head, 0, 0, *tail) if view else lib.ovc_lstm_head(*head, *tail))


kernels = {"k7_one_view": lambda: e.encoded_linear_view(sp._wt0, sp._b0, 0, out=agent._act0),
           "k7_two_views": lambda: e.encoded_linear(sp._wt0, sp._b0, out=sp._act0),
           "k9_n_rows": lambda: k9(agent._act0, agent._z), "k9_2n_rows": lambda: k9(sp._act0, sp._z),
           "k8_view_n_rows": lambda: k8(agent._z, True), "k8_2n_rows": lambda: k8(sp._z, False),
           "k11_view_n_rows": lambda: k11(x1, h1, c1, True), "k11_2n_rows": lambda: k11(x2, h2, c2, False)}
for f in kernels.values():
    f()
torch.cuda.synchronize()
for k, f in kernels.items():
    out[k + "_us"] = min(ms(f, reps=50) for _ in range(3)) * 1e3

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_agent_pair.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
