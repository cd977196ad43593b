#!/usr/bin/env python
"""Cost of population play at the config-5 shape (cramped_room, 32 768 envs), with CUDA events, written as one JSON file
under --out:

  collect(T) for self-play, for a population of self-play learners on blocks (K = 2, 4, 8, 16), for diagonal pairs on the
  same blocks (the cost of the row-grouped path over the blocks path) and for uniform pair_weights; alternated in one
  process, 3 times each;
  run(T) of the evaluation form at K = 2: fixed cross pairs, N / K^2 environments per ordered pair, against one
  AgentPairRollout per ordered pair on N / K^2 environments each, replayed back to back;
  per-kernel times inside CUDA graphs: ovc_group_pairs and ovc_assign_pairs (every environment drawn) on uniform random
  pairs, the grouped masked K7 and the grouped joint K8 on those pairs against the grouped K7 / K8 on equal blocks;
  the card's name and power limit, read in the same run.

    python tools/prof_population_play.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200 import _native  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN, SelfPlayRollout, pair_thresholds  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--ks", default="2,4,8,16")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_population_play measures on a CUDA device"


def ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def graph_us(fn, calls=20):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(calls):
            fn()
    g.replay()
    torch.cuda.synchronize()
    reps = [ms(g.replay) * 1e3 / calls for _ in range(5)]
    return {"min": min(reps), "max": max(reps)}


N, T, KS = args.n, args.steps, [int(k) for k in args.ks.split(",")]
torch.manual_seed(0)
models = [RllibShapedCNN(5, 4).cuda() for _ in range(max(KS))]
env = lambda n: BatchedOvercookedEnv(["cramped_room"], n, horizon=400, auto_reset=True)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)", "kernel_us": {}, "collect_ms": {}, "run_ms": {}}
lib = _native.lib()
st = lambda: torch.cuda.current_stream().cuda_stream

# ---- kernels on uniform random pairs, against the grouped K7 / K8 on equal blocks of the same rows
rows = 2 * N
kenv = env(N)
i32 = lambda n: torch.empty(n, dtype=torch.int32, device="cuda")
a0 = torch.empty(rows, 512, dtype=torch.bfloat16, device="cuda")
x = (torch.randn(rows, 160, device="cuda") * 0.5).to(torch.bfloat16)
acts, vals, logp = i32(rows), torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
counter, pcounter = torch.zeros(2, dtype=torch.int64, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
lst, first, jrow = i32(rows), i32(rows), i32(rows)
for K in KS:
    sp = SelfPlayRollout(env(max(N // 8, K)), models[:K], use_graph=False)
    wt, b0 = sp._learners._k7_stack
    t1, tb1, th, tbh, to, tbo = sp._learners._tail_stack
    pair = torch.randint(0, K, (N, 2), dtype=torch.int32, device="cuda")
    thr = torch.from_numpy(pair_thresholds(np.ones((K, K)), K)).cuda()
    eo, ro = i32(K + 1), i32(K + 1)
    kenv.group_pairs(pair, K, lst, first, jrow, eo, ro)
    boff = torch.tensor([k * N // K for k in range(K + 1)], dtype=torch.int32, device="cuda")
    broff = 2 * boff
    tail = lambda: (t1.data_ptr(), tb1.data_ptr(), th.data_ptr(), tbh.data_ptr(), th.shape[1], to.data_ptr(), tbo.data_ptr(), 0.3, 6, 1,
                    counter.data_ptr())
    fns = {
        "group_pairs": lambda: kenv.group_pairs(pair, K, lst, first, jrow, eo, ro),
        "assign_pairs": lambda: kenv.assign_pairs(pair, K, thr, pcounter, seed=5),
        "grouped_masked_k7": lambda: _native.check(lib.ovc_encode_linear_grouped_masked(
            kenv.tables.data_ptr(), 1, kenv.state.data_ptr(), lst.data_ptr(), first.data_ptr(), wt.data_ptr(), b0.data_ptr(), eo.data_ptr(), K,
            a0.data_ptr(), rows, kenv.state_words, 5, 4, 400, 512, 0.2, st())),
        "grouped_k7_blocks": lambda: _native.check(lib.ovc_encode_linear_grouped(
            kenv.tables.data_ptr(), 1, kenv.state.data_ptr(), wt.data_ptr(), b0.data_ptr(), boff.data_ptr(), K, a0.data_ptr(), N,
            kenv.state_words, 5, 4, 400, 512, 0.2, st())),
        "grouped_joint_k8": lambda: _native.check(lib.ovc_policy_tail_grouped_joint(
            x.data_ptr(), rows, 160, 0.2, *tail(), jrow.data_ptr(), ro.data_ptr(), K, acts.data_ptr(), vals.data_ptr(), 0, logp.data_ptr(),
            st())),
        "grouped_k8_blocks": lambda: _native.check(lib.ovc_policy_tail_grouped(
            x.data_ptr(), rows, 160, 0.2, *tail(), broff.data_ptr(), K, acts.data_ptr(), vals.data_ptr(), 0, logp.data_ptr(), st())),
    }
    out["kernel_us"]["K%d" % K] = {k: graph_us(f) for k, f in fns.items()}
    print("K%d" % K, {k: round(v["min"], 1) for k, v in out["kernel_us"]["K%d" % K].items()}, flush=True)
    del sp
del x, a0, acts, vals, logp, kenv


def alternate(runs, call, reps=3):
    for rs in runs.values():
        for r in rs:
            call(r)  # capture + warm
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(reps):
        for k, rs in runs.items():
            times[k].append(ms(lambda: [call(r) for r in rs]))
    return {k: {"min": min(v), "max": max(v), "all": v} for k, v in times.items()}


# ---- collect(T): one group of rollouts per K, alternated with self-play
col = lambda r: r.collect(T, 0.99, 0.98)
single = SelfPlayRollout(env(N), models[0], seed=1)
for K in KS:
    member = torch.repeat_interleave(torch.arange(K, device="cuda"), N // K).to(torch.int32)
    diag = torch.stack([member, member], 1).contiguous()
    runs = {"self_play": [single], "blocks_k%d" % K: [SelfPlayRollout(env(N), models[:K], seed=1)],
            "diagonal_pairs_k%d" % K: [SelfPlayRollout(env(N), models[:K], pairs=diag, seed=1)],
            "uniform_pair_weights_k%d" % K: [SelfPlayRollout(env(N), models[:K], pair_weights=np.ones((K, K)), seed=1)]}
    res = alternate(runs, col)
    out["collect_ms"]["self_play_with_k%d" % K] = res.pop("self_play")
    out["collect_ms"].update(res)
    for k, v in res.items():
        print(k, "%.2f ms (%.2f - %.2f)" % (v["min"], v["min"], v["max"]), flush=True)
    del runs, res
    torch.cuda.empty_cache()
del single

# ---- the evaluation form at K = 2: fixed cross pairs against one AgentPairRollout per ordered pair
K = 2
q = N // (K * K)
pairs = torch.tensor([(i, j) for i in range(K) for j in range(K)], dtype=torch.int32, device="cuda").repeat_interleave(q, 0).contiguous()
runs = {"fixed_pairs_k2": [SelfPlayRollout(env(K * K * q), models[:K], pairs=pairs, seed=1)],
        "agent_pairs_k2": [AgentPairRollout(env(q), (models[i], models[j]), seed=1) for i in range(K) for j in range(K)]}
out["run_ms"] = alternate(runs, lambda r: r.run(T))
for k, v in out["run_ms"].items():
    print(k, "%.2f ms (%.2f - %.2f)" % (v["min"], v["min"], v["max"]), flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "prof_population_play.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps({k: v for k, v in out.items() if k != "kernel_us"}))
