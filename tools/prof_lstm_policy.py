#!/usr/bin/env python
"""Cost of the LSTM PPO policy (RllibLSTMShapedCNN) at the config-5 shape (cramped_room, 32 768 envs = 65 536 rows,
T = 400), with CUDA events, written as one JSON file under --out:

  K11 (ovc_lstm_head) alone at 65 536 rows, 50 launches, best of 3, with achieved FLOP/s and bytes/s against the bounds
  computed from shapes (0.66 MFLOP and 3 212 bytes per row; 989 TFLOP/s dense bf16 and 3.35 TB/s from the H100 SXM data
  sheet);
  K8's hidden output (ovc_policy_hidden) the same way;
  collect(T) with RllibShapedCNN and with RllibLSTMShapedCNN, alternated in one process, 3 times each;
  the card's name and power limit, read in the same run.

    python tools/prof_lstm_policy.py --out DIR
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
from overcooked_ai_b200.selfplay import RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_lstm_policy measures on a CUDA device"


def ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


N, T = args.n, args.steps
rows = 2 * N
torch.manual_seed(0)
sps = {"cnn": SelfPlayRollout(BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True), model=RllibShapedCNN(5, 4), seed=1),
       "lstm": SelfPlayRollout(BatchedOvercookedEnv(["cramped_room"], N, horizon=400, auto_reset=True), model=RllibLSTMShapedCNN(5, 4), seed=1)}
assert all(sp.fused_first_layer and sp.fused_wide and sp.fused_tail for sp in sps.values())
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "rows": rows, "steps": T, "layout": "cramped_room",
       "policies": {"cnn": "K7 -> K9 -> K8", "lstm": "K7 -> K9 -> K8 hidden -> K11 (LSTM 256)"}}

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
out["collect_lstm_over_cnn"] = min(times["lstm"]) / min(times["cnn"])

sp = sps["lstm"]
lib = _native.lib()
w, b, wo, bo = sp._lstm_tables
w1, b1, wh, bh = sp._tail
h2, c2 = torch.empty_like(sp.h), torch.empty_like(sp.c)
acts = torch.empty(rows, dtype=torch.int32, device="cuda")
vals, logp = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
sp.h.normal_(), sp.c.normal_(), sp._x.normal_()


def k11():
    _native.check(lib.ovc_lstm_head(sp._x.data_ptr(), sp.h.data_ptr(), sp.c.data_ptr(), sp.env.done.data_ptr(), rows, w.data_ptr(),
                                    b.data_ptr(), wo.data_ptr(), bo.data_ptr(), 6, 7, counter.data_ptr(), h2.data_ptr(), c2.data_ptr(), 0, 0,
                                    acts.data_ptr(), vals.data_ptr(), logp.data_ptr(), 0, 0))


def k8_hidden():
    _native.check(lib.ovc_policy_hidden(sp._z.data_ptr(), rows, sp._z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(),
                                        bh.data_ptr(), wh.shape[0], 0.2, sp._x.data_ptr(), 0))


for f in (k11, k8_hidden):
    f()
torch.cuda.synchronize()
t11 = min(ms(k11, reps=50) for _ in range(3)) * 1e-3  # seconds
flop, byts = 2.0 * rows * 1024 * 320 + 2.0 * rows * 8 * 256, rows * (64 * 2 + 256 * 2 * 2 + 256 * 4 * 2 + 12)
out["k11_us"] = t11 * 1e6
out["k11_flop"], out["k11_bytes"] = flop, byts
out["k11_tflops"], out["k11_tb_per_s"] = flop / t11 / 1e12, byts / t11 / 1e12
out["k11_bound_us"] = {"compute_989_tflops": flop / 989e12 * 1e6, "hbm_3.35_tbps": byts / 3.35e12 * 1e6}
out["k11_share_of_hbm_bound"] = byts / 3.35e12 / t11
out["k8_hidden_us"] = min(ms(k8_hidden, reps=50) for _ in range(3)) * 1e3

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_lstm_policy.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
