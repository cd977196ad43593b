#!/usr/bin/env python
"""Cost of collecting PPO sample batches at the config-5 shape (cramped_room, 32 768 envs, K7 -> K9 -> K8 -> K1, T = 400),
with CUDA events, written as one JSON file under --out:

  run(T) against collect(T), alternated in one process, 3 times each (collect adds the record copy, the logp / reward /
  done outputs, the bootstrap evaluation and GAE);
  ovc_gae alone over 20 launches, with the bytes it has to move (T * 2N * 16 + T * N + 2N * 4: rewards and values in,
  advantages and value targets out, the done flags, the bootstrap values) over its time, against the H100 SXM data
  sheet's 3.35 TB/s of HBM3 bandwidth;
  K8 (ovc_policy_tail) with and without the logp output;
  the card's name and power limit, read in the same run.

    python tools/prof_ppo_collect.py --out DIR
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
from overcooked_ai_b200.selfplay import SelfPlayRollout  # noqa: E402

H100_SXM_DATASHEET_HBM_BPS = 3.35e12

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_ppo_collect measures on a CUDA device"


def ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


N, T = args.n, args.steps
env = BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True)
torch.manual_seed(0)
sp = SelfPlayRollout(env, seed=1)
assert sp.fused_first_layer and sp.fused_wide and sp.fused_tail
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T,
       "layout": "cramped_room", "policy": "K7 -> K9 -> K8 (bf16)"}

sp.run(T)  # capture + warm every shape
batch = sp.collect(T, 0.99, 0.95)
torch.cuda.synchronize()
run_ms, collect_ms = [], []
for _ in range(3):
    run_ms.append(ms(lambda: sp.run(T)))
    collect_ms.append(ms(lambda: sp.collect(T, 0.99, 0.95)))
out["run_ms"], out["collect_ms"] = run_ms, collect_ms
out["run_us_per_transition"] = min(run_ms) * 1e3 / T
out["collect_us_per_transition"] = min(collect_ms) * 1e3 / T
out["collect_over_run"] = min(collect_ms) / min(run_ms)

adv, tgt = torch.empty_like(batch.rewards), torch.empty_like(batch.rewards)
gae = lambda: env.gae(batch.rewards, batch.values, batch.dones, batch.last_values, 0.99, 0.95, adv, tgt)  # noqa: E731
gae()
torch.cuda.synchronize()
gae_ms = ms(gae, reps=20)
gae_bytes = T * 2 * N * 16 + T * N + 2 * N * 4
out["gae_us"] = gae_ms * 1e3
out["gae_bytes"] = gae_bytes
out["gae_GBps"] = gae_bytes / (gae_ms * 1e-3) / 1e9
out["gae_share_of_h100_sxm_datasheet_3.35TBps"] = gae_bytes / (gae_ms * 1e-3) / H100_SXM_DATASHEET_HBM_BPS

w1, b1, wh, bh, wo, bo = sp._tail
rows = 2 * N
z = torch.randn((rows, w1.shape[1]), device=env.device).to(torch.bfloat16)
acts = torch.empty(rows, dtype=torch.int32, device=env.device)
vals, logp = torch.empty(rows, dtype=torch.float32, device=env.device), torch.empty(rows, dtype=torch.float32, device=env.device)
counter = torch.zeros(2, dtype=torch.int64, device=env.device)
targs = (z.data_ptr(), rows, z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0], wo.data_ptr(),
         bo.data_ptr(), 0.3, 6, 1, counter.data_ptr(), acts.data_ptr(), vals.data_ptr(), 0)
k8 = lambda: _native.check(_native.lib().ovc_policy_tail(*targs, env._stream()))  # noqa: E731
k8_logp = lambda: _native.check(_native.lib().ovc_policy_tail_logp(*targs, logp.data_ptr(), env._stream()))  # noqa: E731
k8(), k8_logp()
torch.cuda.synchronize()
k8_us, k8_logp_us = [], []
for _ in range(3):
    k8_us.append(ms(k8, reps=50) * 1e3)
    k8_logp_us.append(ms(k8_logp, reps=50) * 1e3)
out["k8_policy_tail_us"], out["k8_policy_tail_logp_us"] = min(k8_us), min(k8_logp_us)

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_ppo_collect.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
