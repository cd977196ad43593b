#!/usr/bin/env python
"""Cost of self-play mixtures at the config-5 shape (cramped_room, 32 768 envs, collect(400)), with CUDA events, written as
one JSON file under --out:

  collect(T) of SelfPlayRollout(PPO); SelfPlayRollout(PPO, partner=frozen PPO) at bc_factor 0, 0.5 and 1;
  AgentPairRollout((PPO, frozen PPO), random_seats=True); SelfPlayRollout(PPO, partner=[4 frozen PPO]) at bc_factor 0.5;
  alternated in one process, 3 times each;
  per-kernel times, best of 3 over 50 launches, at N environments: ovc_learner_rows, the masked K7 and the joint K8 on the
  learner rows of all-self-play (2N rows) and all-paired (N rows) seats, against the two-view K7 and K8 on 2N rows;
  the card's name and power limit, read in the same run.

    python tools/prof_selfplay_mixture.py --out DIR
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
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_selfplay_mixture measures on a CUDA device"


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
ppo = [RllibShapedCNN(5, 4).cuda() for _ in range(4)]
env = lambda: BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)"}
collects = {"selfplay": SelfPlayRollout(env(), learner, seed=1)}
for f in (0.0, 0.5, 1.0):
    collects["mixture_ppo_f%g" % f] = SelfPlayRollout(env(), learner, seed=1, partner=ppo[0], bc_factor=f)
collects["pair_ppo_frozen_ppo"] = AgentPairRollout(env(), (learner, ppo[0]), seed=1, random_seats=True)
collects["mixture_population_ppo_k4_f0.5"] = SelfPlayRollout(env(), learner, seed=1, partner=ppo, bc_factor=0.5)
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
base = min(ctimes["selfplay"])
for k in ctimes:
    out[k + "_over_selfplay"] = min(ctimes[k]) / base

# per-kernel at N environments: the learner's rows of all-self-play and all-paired seats against the two-view kernels
mix = collects["mixture_ppo_f0.5"]
e, lib, s = mix.env, _native.lib(), mix.env._stream()
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
acts = torch.zeros(2 * N, dtype=torch.int32, device="cuda")
vals, logp = torch.zeros(2 * N, device="cuda"), torch.zeros(2 * N, device="cuda")
seats = {"self_play": torch.full((N,), -1, dtype=torch.int32, device="cuda"), "paired": (torch.arange(N, device="cuda") % 2).to(torch.int32)}


def k8(joint):
    w1, b1, wh, bh, wo, bo = mix._tail
    a = (mix._z.data_ptr(), 2 * N, mix._z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0],
         wo.data_ptr(), bo.data_ptr(), 0.3, 6, 1, counter.data_ptr())
    if joint:
        _native.check(lib.ovc_policy_tail_joint(*a, mix._jrow.data_ptr(), mix._lrange.data_ptr(), acts.data_ptr(), vals.data_ptr(), 0,
                                                logp.data_ptr(), s))
    else:
        _native.check(lib.ovc_policy_tail_logp(*a, acts.data_ptr(), vals.data_ptr(), 0, logp.data_ptr(), s))


kernels = {"k7_two_view_2n": lambda: e.encoded_linear(mix._wt0, mix._b0, out=mix._act0),
           "k8_two_view_2n": lambda: k8(False)}
for name, ps in seats.items():
    kernels["learner_rows_" + name] = (lambda ps=ps: e.learner_rows(ps, mix._lst, mix._first, mix._jrow, mix._lrange))
    kernels["k7_masked_" + name] = (lambda ps=ps: (e.learner_rows(ps, mix._lst, mix._first, mix._jrow, mix._lrange),
                                                   e.encoded_linear_masked(mix._wt0, mix._b0, mix._lst, mix._first, mix._act0)))
    kernels["k8_joint_" + name] = (lambda ps=ps: (e.learner_rows(ps, mix._lst, mix._first, mix._jrow, mix._lrange), k8(True)))
for f in kernels.values():
    f()
torch.cuda.synchronize()
for k, f in kernels.items():
    out[k + "_us"] = min(ms(f, reps=50) for _ in range(3)) * 1e3
for name in seats:  # the masked K7 and the joint K8 alone: the scan's time taken out
    out["k7_masked_only_" + name + "_us"] = out["k7_masked_" + name + "_us"] - out["learner_rows_" + name + "_us"]
    out["k8_joint_only_" + name + "_us"] = out["k8_joint_" + name + "_us"] - out["learner_rows_" + name + "_us"]

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_selfplay_mixture.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
