#!/usr/bin/env python
"""Cost of the BC partner (PPO_BC) at the config-5 shape (cramped_room, 32 768 envs, T = 400), with CUDA events, written as
one JSON file under --out:

  K10 (ovc_partner_policy) with every environment paired and with none paired, and ovc_assign_partners, each over 50
  launches, best of 3;
  collect(T) with no partner, with a partner at bc_factor = 0 and at bc_factor = 1, alternated in one process, 3 times each;
  the PPO policy alone (K7 -> K9 -> K8 on both seats of every environment): at bc_factor = 1 half of its rows are the
  partner's and their draws are discarded, so half of this time is what evaluating only the learner's rows could save;
  the card's name and power limit, read in the same run.

    python tools/prof_bc_partner.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import BCPolicy, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_bc_partner measures on a CUDA device"


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
model = RllibShapedCNN(5, 4).cuda()
bc = BCPolicy().cuda()
envs = [BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True) for _ in range(3)]
sps = {"no_partner": SelfPlayRollout(envs[0], model=model, seed=1),
       "bc_factor_0": SelfPlayRollout(envs[1], model=model, seed=1, partner=bc, bc_factor=0.0),
       "bc_factor_1": SelfPlayRollout(envs[2], model=model, seed=1, partner=bc, bc_factor=1.0)}
assert all(sp.fused_first_layer and sp.fused_wide and sp.fused_tail for sp in sps.values())
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)", "partner": "BCPolicy 96 -> 64 -> 64 -> 6 (K10)"}

for sp in sps.values():
    sp.collect(T, 0.99, 0.95)  # capture + warm every shape
torch.cuda.synchronize()
times = {k: [] for k in sps}
for _ in range(3):
    for k, sp in sps.items():
        times[k].append(ms(lambda: sp.collect(T, 0.99, 0.95)))
for k, v in times.items():
    out["collect_ms_" + k] = v
    out["collect_us_per_transition_" + k] = min(v) * 1e3 / T
out["collect_bc_factor_1_over_no_partner"] = min(times["bc_factor_1"]) / min(times["no_partner"])
assert bool((sps["bc_factor_1"].partner_seat >= 0).all())

env = envs[0]
tables = bc.tables()
acts = torch.zeros((N, 2), dtype=torch.int32, device="cuda")
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
seat_all, seat_none = (torch.arange(N, dtype=torch.int32, device="cuda") % 2), torch.full((N,), -1, dtype=torch.int32, device="cuda")
factor = torch.full((1,), 0.5, dtype=torch.float32, device="cuda")
seat = seat_all.clone()
kernels = {"k10_all_paired": lambda: env.partner_actions(tables, seat_all, counter, seed=3, out=acts),
           "k10_none_paired": lambda: env.partner_actions(tables, seat_none, counter, seed=3, out=acts),
           "assign_partners": lambda: env.assign_partners(seat, factor, counter, seed=4, done=env.done),
           "ppo_policy_both_seats": lambda: sps["no_partner"]._policy()}
for f in kernels.values():
    f()
torch.cuda.synchronize()
for k, f in kernels.items():
    out[k + "_us"] = min(ms(f, reps=50) for _ in range(3)) * 1e3

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_bc_partner.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
