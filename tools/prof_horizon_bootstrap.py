#!/usr/bin/env python
"""Cost of collect(bootstrap_horizon=True) at the config-5 shape (cramped_room, 32 768 envs, T = 400, horizon 400), with
CUDA events, written as one JSON file under --out:

  collect(T) with and without the flag, for self-play (SelfPlayRollout, K7 -> K9 -> K8) and for (PPO, BC)
  (AgentPairRollout, random seats), alternated in one process, --reps times each;
  the value pass alone (ovc_horizon_rows, K7's rows form, K9's range form, K8's joint form) with no environment done (the
  empty launches every transition pays) and with every environment done (the pass an episode end pays), and
  ovc_horizon_rows alone with none done, each as 50 launches in one CUDA graph, best of 3;
  the card's name and power limit, read in the same run.

    python tools/prof_horizon_bootstrap.py --out DIR
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
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_horizon_bootstrap measures on a CUDA device"


def ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def graphed_us(fn, n=50):
    """Microseconds per call of ``fn``, 50 calls in one CUDA graph (the host's enqueue cost stays out), best of 3."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    return min(ms(g.replay) for _ in range(3)) * 1e3 / n


N, T = args.n, args.steps
torch.manual_seed(0)
model = RllibShapedCNN(5, 4).cuda()
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "horizon": 400,
       "layout": "cramped_room", "learner": "K7 -> K9 -> K8 (bf16)", "partner": "BCPolicy 96 -> 64 -> 64 -> 6 (K10), random seats"}
mk = lambda: BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
rollouts = {"selfplay": SelfPlayRollout(mk(), model=model, seed=1),
            "ppo_bc": AgentPairRollout(mk(), (model, BCPolicy().cuda()), seed=1, random_seats=True)}
for r in rollouts.values():  # capture + warm every shape
    for flag in (False, True):
        r.collect(T, 0.99, 0.95, bootstrap_horizon=flag)
torch.cuda.synchronize()
times = {(k, f): [] for k in rollouts for f in (False, True)}
for _ in range(args.reps):
    for k, r in rollouts.items():
        for f in (False, True):
            times[(k, f)].append(ms(lambda: r.collect(T, 0.99, 0.95, bootstrap_horizon=f)))
for (k, f), v in times.items():
    out["collect_ms_%s%s" % (k, "_bootstrap" if f else "")] = v
for k in rollouts:
    out["collect_bootstrap_over_plain_%s" % k] = min(times[(k, True)]) / min(times[(k, False)])

# the value pass alone, on the states collect() left (mid-episode: no environment done) and with every environment done
for k, r in rollouts.items():
    learner = r if k == "selfplay" else r.agents[0]
    seats, one_view = (None, False) if k == "selfplay" else (r.partner_seat, True)
    h, env = r._horizon, r.env
    assert h.fused
    vals = torch.empty(h.logp.shape, device="cuda")
    value_pass = lambda: learner._horizon_values_rows(h, seats, one_view, vals, r._boot_counter, r._boot_actions)
    done = env.done.clone()
    env.done.zero_()
    out["value_pass_none_done_us_%s" % k] = graphed_us(value_pass)
    out["horizon_rows_none_done_us_%s" % k] = graphed_us(lambda: env.horizon_rows(seats, one_view, h.records, h.view, h.jrow, h.range, vals))
    env.done.fill_(1)
    out["value_pass_all_done_us_%s" % k] = graphed_us(value_pass)
    env.done.copy_(done)

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_horizon_bootstrap.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
