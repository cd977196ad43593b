#!/usr/bin/env python
"""Cost of a population of partners at the config-5 shape (cramped_room, 32 768 envs, collect(400)), with CUDA events,
written as one JSON file under --out:

  collect(T) of AgentPairRollout(PPO, [K frozen PPO members]) with random seats and uniformly drawn members for K = 1, 2, 4,
  8, against the pair (PPO, frozen PPO); AgentPairRollout(PPO, [4 BC members]) against the pair (PPO, BC); alternated in
  one process, 3 times each;
  per-kernel times, best of 3 over 50 launches: ovc_group_members and ovc_assign_members at N environments (K = 8), and
  each rows form on N / K rows against its one-view form on N / K rows (K = 8);
  the card's name and power limit, read in the same run.

    python tools/prof_population.py --out DIR
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
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN, member_thresholds  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_population measures on a CUDA device"


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
learner = RllibShapedCNN(5, 4).cuda()
ppo = [RllibShapedCNN(5, 4).cuda() for _ in range(8)]
bcs = [BCPolicy().cuda() for _ in range(4)]
env = lambda: BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)", "bc": "BCPolicy 96 -> 64 -> 64 -> 6 (K10)"}
collects = {"pair_ppo_frozen_ppo": AgentPairRollout(env(), (learner, ppo[0]), seed=1, random_seats=True)}
for k in (1, 2, 4, 8):
    collects["population_ppo_k%d" % k] = AgentPairRollout(env(), (learner, ppo[:k]), seed=1, random_seats=True)
collects["pair_ppo_bc"] = AgentPairRollout(env(), (learner, bcs[0]), seed=1, random_seats=True)
collects["population_bc_k4"] = AgentPairRollout(env(), (learner, bcs), seed=1, random_seats=True)
for r in collects.values():
    r.collect(T, 0.99, 0.98)  # capture + warm
torch.cuda.synchronize()
ctimes = {k: [] for k in collects}
for _ in range(3):
    for k, r in collects.items():
        ctimes[k].append(ms(lambda: r.collect(T, 0.99, 0.98)))
for k, v in ctimes.items():
    out["collect_ms_" + k] = v
    out["collect_us_per_transition_" + k] = min(v) * 1e3 / T
base = min(ctimes["pair_ppo_frozen_ppo"])
for k in (1, 2, 4, 8):
    out["population_ppo_k%d_over_pair" % k] = min(ctimes["population_ppo_k%d" % k]) / base
out["population_bc_k4_over_pair"] = min(ctimes["population_bc_k4"]) / min(ctimes["pair_ppo_bc"])

# per-kernel, K = 8: the two population kernels at N environments, each rows form on N / K rows against its one-view form
pop = collects["population_ppo_k8"]
P = pop.agents[1]
e = pop.env
lib, s = _native.lib(), e._stream()
K = 8
thr = torch.from_numpy(member_thresholds([1.0] * K)).cuda()
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
member = (torch.arange(N, device="cuda") % K).to(torch.int32)
order, offsets = torch.empty(N, dtype=torch.int32, device="cuda"), torch.empty(K + 1, dtype=torch.int32, device="cuda")
e.group_members(member, K, order, offsets)
rng = offsets[3:5]  # one member's share: N / K rows from an unaligned start
Nk = N // K
net = P.agents[0]
env_k = BatchedOvercookedEnv(["cramped_room"], Nk, horizon=400, auto_reset=True)  # the one-view forms on N / K environments
acts = torch.zeros((N, 2), dtype=torch.int32, device="cuda")
act0_k = torch.empty((Nk, net._wt0.shape[1]), dtype=torch.bfloat16, device="cuda")
z_k = torch.empty((Nk, net._z.shape[1]), dtype=torch.bfloat16, device="cuda")
scores = torch.randn(N, 8, device="cuda")


def k9(a0, m, z, range_=None):
    w1, b1, w2, b2 = net._wide
    args_ = (a0.data_ptr(), m, a0.shape[1], w1.data_ptr(), b1.data_ptr(), w1.shape[0], w2.data_ptr(), b2.data_ptr(), w2.shape[0], 0.2)
    if range_ is None:
        _native.check(lib.ovc_wide_layers(*args_, z.data_ptr(), s))
    else:
        _native.check(lib.ovc_wide_layers_range(*args_, range_.data_ptr(), z.data_ptr(), s))


def k8(z, m, rows=None):
    w1, b1, wh, bh, wo, bo = net._tail
    a = (z.data_ptr(), m, z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0], wo.data_ptr(),
         bo.data_ptr(), 0.3, 6, 1, counter.data_ptr())
    if rows is None:
        _native.check(lib.ovc_policy_tail_view(*a, 0, 0, acts.data_ptr(), 0, 0, 0, s))
    else:
        _native.check(lib.ovc_policy_tail_rows(*a, 0, 0, order.data_ptr(), rng.data_ptr(), acts.data_ptr(), 0, 0, 0, s))


kernels = {"group_members_n_k8": lambda: e.group_members(member, K, order, offsets),
           "assign_members_n_k8": lambda: e.assign_members(member, K, thr, counter, seed=1, done=e.done),
           "k7_rows_n_over_k": lambda: e.encoded_linear_rows(net._wt0, net._b0, 0, None, order, rng, net._act0),
           "k7_one_view_n_over_k": lambda: env_k.encoded_linear_view(net._wt0, net._b0, 0, out=act0_k),
           "k9_range_n_over_k": lambda: k9(net._act0, N, net._z, rng),
           "k9_n_over_k_rows": lambda: k9(act0_k, Nk, z_k),
           "k8_rows_n_over_k": lambda: k8(net._z, N, rows=True),
           "k8_view_n_over_k": lambda: k8(z_k, Nk),
           "sample_rows_n_over_k": lambda: e.sample_actions_rows(scores, counter, 0, None, order, rng, out=acts),
           "sample_view_n_over_k": lambda: env_k.sample_actions_view(scores[:Nk], counter, 0, out=acts[:Nk])}
for f in kernels.values():
    f()
torch.cuda.synchronize()
for k, f in kernels.items():
    out[k + "_us"] = min(ms(f, reps=50) for _ in range(3)) * 1e3

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_population.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
