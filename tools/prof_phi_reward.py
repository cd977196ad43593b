#!/usr/bin/env python
"""Cost of the potential-based dense reward (use_phi) at the config-5 shape (cramped_room, 32 768 envs, collect(400)),
written as one JSON file under --out:

  default      collect(T) of SelfPlayRollout(PPO) and AgentPairRollout((PPO, BC), random_seats=True), each with and without
               use_phi, alternated in one process, 3 times each, timed with CUDA events;
  --kernels    (a separate run: tracing slows the host) torch.profiler's device time per launch of K6 (potential_kernel),
               ovc_potential_shaping and ovc_record_transition_dense, with K1 and the two-row record kernel beside them,
               over one collect(T) of each use_phi rollout;
  the card's name and power limit, read in the same run.

    python tools/prof_phi_reward.py --out DIR [--kernels]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--kernels", action="store_true")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_phi_reward measures on a CUDA device"


def ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


N, T = args.n, args.steps
torch.manual_seed(0)
learner, bc = RllibShapedCNN(5, 4).cuda(), BCPolicy().cuda()
env = lambda: BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)"}
collects = {}
for phi in (False, True):
    tag = "_phi" if phi else ""
    collects["selfplay" + tag] = SelfPlayRollout(env(), learner, seed=1, use_phi=phi)
    collects["pair_ppo_bc" + tag] = AgentPairRollout(env(), (learner, bc), seed=1, random_seats=True, use_phi=phi)
for r in collects.values():
    r.collect(T, 0.99, 0.98)  # capture + warm
torch.cuda.synchronize()

if not args.kernels:
    ctimes = {k: [] for k in collects}
    for _ in range(3):
        for k, r in collects.items():
            ctimes[k].append(ms(lambda: r.collect(T, 0.99, 0.98)))
    for k, v in ctimes.items():
        out["collect_ms_" + k] = v
        out["collect_us_per_transition_" + k] = min(v) * 1e3 / T
    for k in ("selfplay", "pair_ppo_bc"):
        out[k + "_phi_over_plain"] = min(ctimes[k + "_phi"]) / min(ctimes[k])
        out[k + "_phi_extra_us_per_transition"] = (min(ctimes[k + "_phi"]) - min(ctimes[k])) * 1e3 / T
else:
    from torch.profiler import ProfilerActivity, profile

    names = {"potential_kernel": "k6_potential", "potential_shaping_kernel": "potential_shaping",
             "record_transition_dense_kernel": "record_transition_dense", "step_kernel": "k1_step",
             "accumulate_returns_kernel": "record_transition_two_rows"}
    for k in ("selfplay_phi", "pair_ppo_bc_phi", "selfplay"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            collects[k].collect(T, 0.99, 0.98)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            for frag, short in names.items():
                if frag in ev.key and ev.count:
                    dev_us = getattr(ev, "device_time_total", None)
                    dev_us = ev.cuda_time_total if dev_us is None else dev_us
                    out["%s_%s_us_per_launch" % (k, short)] = dev_us / ev.count
                    out["%s_%s_launches" % (k, short)] = ev.count

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_phi_reward%s.json" % ("_kernels" if args.kernels else ""))
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
