#!/usr/bin/env python
"""Seconds per epoch of behaviour-cloning training (include/ovc_bc.h) for K = 1, 4, 16, 64 and 132 models on one dataset,
the reference's five recorded GreedyHumanModel games on cramped_room (tests/golden/greedy_cramped_room.npz: 4 000 rows,
3 400 training rows, 54 minibatches of 64 per epoch), written as one JSON file under --out:

  train_bc: the whole epoch as train_bc runs it (the per-model shuffles, one ovc_bc_train_epoch launch, the stats copy
    and the host callbacks), from the time of 1 + E epochs minus that of 1 epoch, over E;
  the kernel alone: one ovc_bc_train_epoch launch with CUDA events, best of 3;
  the torch trainer: the same recipe in float32 eager torch (BCPolicy, torch.optim.Adam(eps=1e-7), cross entropy, the
    shuffle, the validation pass and one host sync per epoch), run model after model;
  the card's name and power limit, read in the same run.

    python tools/prof_bc_train.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from overcooked_ai_b200 import _bc_native, bc as B  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--models", default="1,4,16,64,132")
ap.add_argument("--epochs", type=int, default=3, help="timed epochs E per measurement")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_bc_train measures on a CUDA device"

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
d = np.load(os.path.join(ROOT, "tests", "golden", "greedy_cramped_room.npz"))
env = BatchedOvercookedEnv("cramped_room", 1, horizon=400)
X, Y = B.bc_dataset(env, d["states"].reshape(-1, 16), d["actions"].reshape(-1, 2))
R, E = X.shape[0], args.epochs
tr_pos, va_pos = B.validation_split_rows(R)
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "rows": R, "train_rows": len(tr_pos),
       "val_rows": len(va_pos), "batch": 64, "network": "96 -> 64 -> 64 -> 6 (10 758 parameters)", "timed_epochs": E, "results": []}


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def train_bc_epoch_s(K):
    run = lambda n: B.train_bc(X, Y, n_models=K, seeds=list(range(K)), epochs=n)  # noqa: E731
    run(1)  # warm-up
    return (wall(lambda: run(1 + E)) - wall(lambda: run(1))) / E


def kernel_ms(K):
    P = B.param_count()
    params = torch.stack([B.glorot_init(k) for k in range(K)]).cuda()
    m, v = torch.zeros_like(params), torch.zeros_like(params)
    step = torch.zeros(K, dtype=torch.int32, device="cuda")
    lr = torch.full((K,), 1e-3, device="cuda")
    active = torch.ones(K, dtype=torch.uint8, device="cuda")
    stats = torch.zeros((K, 4), dtype=torch.float64, device="cuda")
    trows = torch.from_numpy(np.stack([np.random.RandomState(k).permutation(tr_pos) for k in range(K)]).astype(np.int32)).cuda()
    vrows = torch.from_numpy(np.tile(va_pos, (K, 1)).astype(np.int32)).cuda()
    vrows = torch.nn.functional.pad(vrows, (0, trows.shape[1] - vrows.shape[1])).contiguous()
    nt = torch.full((K,), len(tr_pos), dtype=torch.int32, device="cuda")
    nv = torch.full((K,), len(va_pos), dtype=torch.int32, device="cuda")
    lib = _bc_native.lib()
    call = lambda: _bc_native.check(lib.ovc_bc_train_epoch(  # noqa: E731
        X.data_ptr(), Y.data_ptr(), R, trows.data_ptr(), nt.data_ptr(), vrows.data_ptr(), nv.data_ptr(), trows.shape[1], params.data_ptr(),
        m.data_ptr(), v.data_ptr(), step.data_ptr(), lr.data_ptr(), active.data_ptr(), stats.data_ptr(), K, 96, 64, 2, 6, 64,
        torch.cuda.current_stream().cuda_stream))
    assert params.shape[1] == P
    call()
    best = float("inf")
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def torch_epoch_s(K):
    """K models trained one after the other with the recipe in eager float32 torch; seconds per epoch of all K."""
    tr, va = torch.from_numpy(tr_pos).cuda(), torch.from_numpy(va_pos).cuda()
    Yl = Y.long()
    models = []
    for k in range(K):
        pol = B.policy_from_flat(B.glorot_init(k).cuda())
        models.append((pol, torch.optim.Adam(pol.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-7)))

    def epoch(pol, opt):
        perm = tr[torch.randperm(len(tr), device="cuda")]
        tot = torch.zeros((), device="cuda")
        for r0 in range(0, len(perm), 64):
            idx = perm[r0:r0 + 64]
            loss = F.cross_entropy(pol(X[idx]), Yl[idx])
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            tot += loss.detach() * len(idx)
        with torch.no_grad():
            vl = F.cross_entropy(pol(X[va]), Yl[va], reduction="sum")
        return float(tot), float(vl)  # the host sync the callbacks need

    epoch(*models[0])  # warm-up
    return wall(lambda: [epoch(*mo) for _ in range(E) for mo in models]) / E


for K in [int(k) for k in args.models.split(",")]:
    res = {"models": K, "train_bc_s_per_epoch": train_bc_epoch_s(K), "kernel_ms_per_epoch": kernel_ms(K), "torch_s_per_epoch": torch_epoch_s(K)}
    res["speedup_over_torch"] = res["torch_s_per_epoch"] / res["train_bc_s_per_epoch"]
    out["results"].append(res)
    print(json.dumps(res), flush=True)

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_bc_train.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
