#!/usr/bin/env python
"""Launch one kernel family a few times so a profiler (Nsight Compute) can capture it.
    ncu --set full --clock-control none --import-source on -k regex:<name> -s 2 -c 1 -o out python tools/prof_kernels.py --which k5
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--which", default="k5", choices=["k1", "k5", "k2", "k2u8", "k3", "k6", "k7", "k8"])
ap.add_argument("--n", type=int, default=65536)
ap.add_argument("--layouts", default="cramped_room")
ap.add_argument("--reps", type=int, default=4)
args = ap.parse_args()
env = BatchedOvercookedEnv(args.layouts.split(","), args.n, horizon=400, auto_reset=True)
T = 400
acts = torch.randint(0, 6, (T, args.n, 2), dtype=torch.int32, device="cuda")
if args.which == "k5":
    out = env.rollout(acts)
    for _ in range(args.reps):
        env.rollout(acts, out=out)
elif args.which == "k1":
    for t in range(40):
        env.step(acts[t])
elif args.which in ("k7", "k8"):  # the config-5 policy kernels: a few eager self-play transitions (ncu: -k regex:encode_linear|policy_tail)
    from overcooked_ai_b200.selfplay import SelfPlayRollout
    env.rollout(acts[:150])
    sp = SelfPlayRollout(env, use_graph=False)
    for _ in range(args.reps):
        sp._transition()
else:
    env.rollout(acts[:150])
    if args.which == "k6":
        o = env.potential(0.99)
        for _ in range(args.reps):
            env.potential(0.99, out=o)
    elif args.which == "k3":
        o = env.featurize_state(2)
        for _ in range(args.reps):
            env.featurize_state(2, out=o)
    else:
        o = env.lossless_state_encoding(dtype=torch.uint8 if args.which == "k2u8" else torch.float32)
        for _ in range(args.reps):
            env.lossless_state_encoding(out=o)
torch.cuda.synchronize()
print("done", args.which)
