#!/usr/bin/env python
"""Cost of the greedy partner (GreedyHumanModel, include/ovc_greedy.h) at the config-5 shape (cramped_room, 32 768 envs,
T = 400), with CUDA events, written as one JSON file under --out:

  ovc_greedy_actions alone with every environment played (on states reached by a greedy pair, so pots cook and soups are
  carried) and with none played, each as 50 launches in one CUDA graph, best of 3;
  AgentPairRollout run(T) and collect(T) for (PPO, Greedy) against (PPO, BC), random seats, alternated in one process,
  3 times each;
  the card's name and power limit, read in the same run.

    python tools/prof_greedy.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.greedy import GreedyHumanModel  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_greedy measures on a CUDA device"


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
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "learner": "K7 -> K9 -> K8 (bf16)", "partners": {"greedy": "GreedyHumanModel (ovc_greedy_actions)",
                                                         "bc": "BCPolicy 96 -> 64 -> 64 -> 6 (K10)"}}

# the kernel alone, on states a greedy pair reaches
env = BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
warm = AgentPairRollout(env, (GreedyHumanModel(), GreedyHumanModel()), seed=2, use_graph=False)
warm.run(150)
acts = torch.zeros((N, 2), dtype=torch.int32, device="cuda")
prev = torch.zeros(N, dtype=torch.int32, device="cuda")
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
all_played = (torch.arange(N, dtype=torch.int32, device="cuda") % 2)
none_played = torch.full((N,), -1, dtype=torch.int32, device="cuda")
kernels = {"greedy_all_played": lambda: env.greedy_actions(all_played, prev, counter, seed=3, done=env.done, out=acts),
           "greedy_none_played": lambda: env.greedy_actions(none_played, prev, counter, seed=3, done=env.done, out=acts)}
for k, f in kernels.items():  # 50 launches in one CUDA graph, so the host's enqueue cost stays out of the time
    f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(50):
            f()
    g.replay()
    out[k + "_us"] = min(ms(g.replay) for _ in range(3)) * 1e3 / 50

pairs = {"ppo_greedy": AgentPairRollout(BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True),
                                        (model, GreedyHumanModel()), seed=1, random_seats=True),
         "ppo_bc": AgentPairRollout(BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True),
                                    (model, BCPolicy().cuda()), seed=1, random_seats=True)}
for p in pairs.values():  # capture + warm every shape
    p.run(T)
    p.collect(T, 0.99, 0.95)
torch.cuda.synchronize()
times = {(k, w): [] for k in pairs for w in ("run", "collect")}
for _ in range(3):
    for k, p in pairs.items():
        times[(k, "run")].append(ms(lambda: p.run(T)))
        times[(k, "collect")].append(ms(lambda: p.collect(T, 0.99, 0.95)))
for (k, w), v in times.items():
    out["%s_ms_%s" % (w, k)] = v
for w in ("run", "collect"):
    out["%s_greedy_over_bc" % w] = min(times[("ppo_greedy", w)]) / min(times[("ppo_bc", w)])

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_greedy.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
