#!/usr/bin/env python
"""K8 at every first-layer width k0 = 32 .. 256, with CUDA events, written as one JSON file under --out:

  each drawing form of ovc_policy_tail at the config-5 row counts (32 768 environments): the two-view form with and
  without logp on 2N rows; the one-view, rows and joint forms on N rows; the grouped form on 2N rows in 4 equal blocks.
  Each form runs inside a CUDA graph of 20 calls, and the best of 3 replays is kept.  n_hidden = 2 and 6 actions, as in the
  reference's PPO network.  The card's name and power limit are read in the same run.

    python tools/prof_policy_tail.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200 import _native  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--k0", default="32,64,96,128,160,192,224,256")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_policy_tail measures on a CUDA device"

lib = _native.lib()
N, H, A, K = args.n, 2, 6, 4
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "n_hidden": H, "n_actions": A, "us": {}}
torch.manual_seed(0)
dev = "cuda"
i32 = lambda t: torch.tensor(t, dtype=torch.int32, device=dev)
acts, vals, logp = torch.empty(2 * N, dtype=torch.int32, device=dev), torch.empty(2 * N, device=dev), torch.empty(2 * N, device=dev)
counter = torch.zeros(2, dtype=torch.int64, device=dev)
swap = torch.zeros(N, dtype=torch.int32, device=dev)
e = torch.arange(N, dtype=torch.int32, device=dev)
rows, jrow, rng = e, 2 * e + (e & 1), i32([0, N])
offsets = i32([k * 2 * N // K for k in range(K + 1)])
st = lambda: torch.cuda.current_stream().cuda_stream


def graph_us(fn, calls=20):
    fn()
    torch.cuda.synchronize()
    g, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(calls):
            fn()
    best = float("inf")
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3 / calls)
    return best


for k0 in [int(k) for k in args.k0.split(",")]:
    x = (torch.randn(2 * N, k0, device=dev) * 0.5).to(torch.bfloat16)
    w1 = (torch.randn(K, 64, k0, device=dev) * 0.1).to(torch.bfloat16)
    wh = (torch.randn(K, H, 64, 64, device=dev) * 0.1).to(torch.bfloat16)
    wo = (torch.randn(K, 8, 64, device=dev) * 0.1).to(torch.bfloat16)
    b1, bh, bo = torch.randn(K, 64, device=dev) * 0.1, torch.randn(K, H, 64, device=dev) * 0.1, torch.randn(K, 8, device=dev) * 0.1
    tables = lambda k=0: (w1[k].data_ptr(), b1[k].data_ptr(), wh[k].data_ptr(), bh[k].data_ptr(), H, wo[k].data_ptr(), bo[k].data_ptr())
    head = lambda n: (x.data_ptr(), n, k0, 0.2) + tables() + (0.3, A, 1, counter.data_ptr())
    outs = (acts.data_ptr(), vals.data_ptr(), 0, logp.data_ptr())
    forms = {
        "two_view": lambda: _native.check(lib.ovc_policy_tail(*head(2 * N), acts.data_ptr(), vals.data_ptr(), 0, st())),
        "two_view_logp": lambda: _native.check(lib.ovc_policy_tail_logp(*head(2 * N), *outs, st())),
        "view_logp": lambda: _native.check(lib.ovc_policy_tail_view(*head(N), swap.data_ptr(), 0, *outs, st())),
        "rows_logp": lambda: _native.check(lib.ovc_policy_tail_rows(*head(N), swap.data_ptr(), 0, rows.data_ptr(), rng.data_ptr(), *outs, st())),
        "joint": lambda: _native.check(lib.ovc_policy_tail_joint(*head(N), jrow.data_ptr(), rng.data_ptr(), *outs, st())),
        "grouped_k4_logp": lambda: _native.check(lib.ovc_policy_tail_grouped(
            x.data_ptr(), 2 * N, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), H, wo.data_ptr(), bo.data_ptr(), 0.3, A,
            1, counter.data_ptr(), offsets.data_ptr(), K, *outs, st())),
    }
    out["us"]["k0_%d" % k0] = {name: graph_us(fn) for name, fn in forms.items()}
    print("k0 %d" % k0, {k: round(v, 2) for k, v in out["us"]["k0_%d" % k0].items()}, flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "prof_policy_tail.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
