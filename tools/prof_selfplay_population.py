#!/usr/bin/env python
"""Cost of a population of self-play learners at the config-5 shape (cramped_room, 32 768 envs, collect(400)), with CUDA
events, written as one JSON file under --out:

  collect(T) of SelfPlayRollout(env, [m_0, ..., m_{K-1}]) on N environments for K = 1, 2, 4, 8, 16, against one
  SelfPlayRollout on N environments and against K SelfPlayRollouts on N / K environments each, replayed back to back
  (what training K self-play agents costs without the population); alternated in one process, 3 times each;
  per-kernel times inside CUDA graphs (as the rollout runs them): each grouped kernel (K7 on N environments, K9 and K8 on
  2N rows, K equal blocks) against K launches of its existing form (ovc_encode_linear_masked, ovc_wide_layers,
  ovc_policy_tail_logp) on the same blocks;
  the card's name and power limit, read in the same run.

    python tools/prof_selfplay_population.py --out DIR
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
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--ks", default="1,2,4,8,16")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_selfplay_population measures on a CUDA device"


def ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


N, T, KS = args.n, args.steps, [int(k) for k in args.ks.split(",")]
torch.manual_seed(0)
models = [RllibShapedCNN(5, 4).cuda() for _ in range(max(KS))]
env = lambda n: BatchedOvercookedEnv(["cramped_room"], n, horizon=400, auto_reset=True)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "policy": "K7 -> K9 -> K8 (bf16)", "collect_ms": {}, "kernel_us": {}}

# ---- kernels: each grouped kernel against K launches of its existing form on the same blocks, both arms captured in CUDA
# graphs (as the rollout runs them), best of 3 replays of 20 calls
lib = _native.lib()
rows = 2 * N
kenv = env(N)
a0 = torch.empty(rows, 512, dtype=torch.bfloat16, device="cuda")
x = (torch.randn(rows, 160, device="cuda") * 0.5).to(torch.bfloat16)
z = torch.empty_like(x)
acts, vals, logp = torch.empty(rows, dtype=torch.int32, device="cuda"), torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
counter = torch.zeros(2, dtype=torch.int64, device="cuda")
e_ = torch.arange(N, dtype=torch.int32, device="cuda")
k7_list, k7_first = (e_ << 2) | 3, 2 * e_


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
    return min(ms(g.replay) for _ in range(3)) * 1e3 / calls


for K in KS:
    sp = SelfPlayRollout(env(max(N // 8, K)), models[:K], use_graph=False)
    wt, b0 = sp._learners._k7_stack
    w1, b1, w2, b2 = sp._learners._wide_stack
    t1, tb1, th, tbh, to, tbo = sp._learners._tail_stack
    eoff = torch.tensor([k * N // K for k in range(K + 1)], dtype=torch.int32, device="cuda")
    roff = 2 * eoff
    ho = eoff.tolist()
    st = lambda: torch.cuda.current_stream().cuda_stream

    def k7_grouped():
        _native.check(lib.ovc_encode_linear_grouped(kenv.tables.data_ptr(), 1, kenv.state.data_ptr(), wt.data_ptr(), b0.data_ptr(),
                                                    eoff.data_ptr(), K, a0.data_ptr(), N, kenv.state_words, 5, 4, 400, 512, 0.2, st()))

    def k7_each():  # the existing two-view form per member on its block (ovc_encode_linear_masked on its list entries)
        for k in range(K):
            a, b = ho[k], ho[k + 1]
            _native.check(lib.ovc_encode_linear_masked(kenv.tables.data_ptr(), 1, kenv.state.data_ptr(), k7_list[a:].data_ptr(),
                                                       k7_first[a:].data_ptr(), wt[k].data_ptr(), b0[k].data_ptr(), a0.data_ptr(), b - a,
                                                       kenv.state_words, 5, 4, 400, 512, 0.2, st()))

    def k9_grouped():
        _native.check(lib.ovc_wide_layers_grouped(a0.data_ptr(), rows, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(),
                                                  160, 0.2, roff.data_ptr(), K, z.data_ptr(), st()))

    def k9_each():
        for k in range(K):
            a, n = 2 * ho[k], 2 * (ho[k + 1] - ho[k])
            _native.check(lib.ovc_wide_layers(a0[a:].data_ptr(), n, 512, w1[k].data_ptr(), b1[k].data_ptr(), 512, w2[k].data_ptr(),
                                              b2[k].data_ptr(), 160, 0.2, z[a:].data_ptr(), st()))

    def k8_grouped():
        _native.check(lib.ovc_policy_tail_grouped(x.data_ptr(), rows, 160, 0.2, t1.data_ptr(), tb1.data_ptr(), th.data_ptr(), tbh.data_ptr(),
                                                  th.shape[1], to.data_ptr(), tbo.data_ptr(), 0.3, 6, 1, counter.data_ptr(), roff.data_ptr(), K,
                                                  acts.data_ptr(), vals.data_ptr(), 0, logp.data_ptr(), st()))

    def k8_each():
        for k in range(K):
            a, n = 2 * ho[k], 2 * (ho[k + 1] - ho[k])
            _native.check(lib.ovc_policy_tail_logp(x[a:].data_ptr(), n, 160, 0.2, t1[k].data_ptr(), tb1[k].data_ptr(), th[k].data_ptr(),
                                                   tbh[k].data_ptr(), th.shape[1], to[k].data_ptr(), tbo[k].data_ptr(), 0.3, 6, 1, counter.data_ptr(),
                                                   acts[a:].data_ptr(), vals[a:].data_ptr(), 0, logp[a:].data_ptr(), st()))

    out["kernel_us"]["K%d" % K] = {"grouped_k7": graph_us(k7_grouped), "k_launches_k7": graph_us(k7_each),
                                   "grouped_k9": graph_us(k9_grouped), "k_launches_k9": graph_us(k9_each),
                                   "grouped_k8": graph_us(k8_grouped), "k_launches_k8": graph_us(k8_each)}
    print("K%d" % K, {k: round(v, 1) for k, v in out["kernel_us"]["K%d" % K].items()}, flush=True)
    del sp
del x, z, a0, acts, vals, logp, kenv

# ---- collect(T): the population, one rollout on N environments, K rollouts on N / K environments
runs = {"single_n": [SelfPlayRollout(env(N), models[0], seed=1)]}
for K in KS:
    runs["population_k%d" % K] = [SelfPlayRollout(env(N), models[:K], seed=1)]
    if K > 1:
        runs["k_rollouts_k%d" % K] = [SelfPlayRollout(env(N // K), m, seed=1) for m in models[:K]]
for rs in runs.values():
    for r in rs:
        r.collect(T, 0.99, 0.98)  # capture + warm
torch.cuda.synchronize()
times = {k: [] for k in runs}
for _ in range(3):
    for k, rs in runs.items():
        times[k].append(ms(lambda: [r.collect(T, 0.99, 0.98) for r in rs]))
out["collect_ms"] = {k: {"min": min(v), "all": v} for k, v in times.items()}
for k, v in out["collect_ms"].items():
    print(k, "%.2f ms" % v["min"], flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "prof_selfplay_population.json"), "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
