#!/usr/bin/env python
"""Kernel micro-benchmarks on one GPU: K1 (each record-I/O strategy), K5, K2, K3 over batch sizes.

Timing: CUDA events around a CUDA-graph replay of `reps` launches (graph removes the Python launch
cost; what is left per launch is kernel time + launch gap).  For batch sizes whose working set fits
the L2 (50 MB on an H100) the numbers are L2-assisted; the 4M-env rows exceed L2 and are HBM-true.
Prints one JSON line per measurement.  Usage: python tools/kbench.py [--layout cramped_room] [--quick]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--layouts", default="cramped_room")
ap.add_argument("--sizes", default="65536,262144,1048576,4194304")
ap.add_argument("--ios", default="1,2,3")
ap.add_argument("--reps", type=int, default=40)
ap.add_argument("--what", default="k1,k5,k2,k3")
ap.add_argument("--pdl", default="0,1")
args = ap.parse_args()
layouts = args.layouts.split(",")
PEAK = 6485.5
if os.path.exists("MEASURED_PEAKS.json"):
    PEAK = json.load(open("MEASURED_PEAKS.json"))["hbm_gbs"]


def time_graph(fn, reps, iters=5):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / reps)
    return best * 1e3  # us per launch


for n in [int(x) for x in args.sizes.split(",")]:
    what = args.what.split(",")
    for io in [int(x) for x in args.ios.split(",")]:
        env = BatchedOvercookedEnv(layouts, n, horizon=400, auto_reset=True, io=io)
        S = env.state_words
        bytes_step = 2 * 4 * S + 32
        # a ring of action tensors so consecutive launches read different actions
        acts = torch.randint(0, 6, (8, n, 2), dtype=torch.int32, device="cuda")
        k = [0]

        def k1():
            env.step(acts[k[0] % 8])
            k[0] += 1

        if "k1" in what:
            for pdl in [int(x) for x in args.pdl.split(",")]:
                env.pdl = bool(pdl)
                us = time_graph(k1, args.reps)
                gbs = n * bytes_step / us / 1e3
                print(json.dumps({"kernel": "K1 step", "io": io, "pdl": pdl, "n_envs": n, "S": S, "us_per_launch": round(us, 3),
                                  "env_steps_per_s": n / us * 1e6, "algorithmic_GBps": round(gbs, 1), "frac_of_measured_hbm": round(gbs / PEAK, 4)}), flush=True)
            env.pdl = False
        if "k5" in what and n <= 1048576:
            T = 50
            ra = torch.randint(0, 6, (T, n, 2), dtype=torch.int32, device="cuda")
            out = env.rollout(ra)

            def k5():
                env.rollout(ra, out=out)

            us = time_graph(k5, 4, iters=3)
            print(json.dumps({"kernel": "K5 rollout T=50", "io": io, "n_envs": n, "S": S, "us_per_launch": round(us, 2),
                              "env_steps_per_s": n * T / us * 1e6, "streamed_GBps": round(n * T * 32 / us / 1e3, 1)}), flush=True)
            del ra, out
        del env, acts
        torch.cuda.empty_cache()
    if n > 1048576:
        continue
    env = BatchedOvercookedEnv(layouts, n, horizon=400, auto_reset=True)
    env.rollout(torch.randint(0, 6, (60, n, 2), dtype=torch.int32, device="cuda"))
    S = env.state_words
    l = env.layouts[0]
    if "k2" in what and len({(x.width, x.height) for x in env.layouts}) == 1:
        for dt, es in ((torch.float32, 4), (torch.uint8, 1)):
            o = env.lossless_state_encoding(dtype=dt)

            def k2():
                env.lossless_state_encoding(out=o)

            us = time_graph(k2, 10)
            b = n * (4 * S + 2 * l.width * l.height * 26 * es)
            print(json.dumps({"kernel": "K2 lossless " + str(dt).split(".")[1], "n_envs": n, "S": S, "us_per_launch": round(us, 2),
                              "encodes_per_s": n / us * 1e6, "algorithmic_GBps": round(b / us / 1e3, 1), "frac_of_measured_hbm": round(b / us / 1e3 / PEAK, 4)}), flush=True)
            del o
    if "k3" in what:
        o = env.featurize_state(2)

        def k3():
            env.featurize_state(2, out=o)

        us = time_graph(k3, 10)
        b = n * (4 * S + 2 * 96 * 4)
        print(json.dumps({"kernel": "K3 featurize", "n_envs": n, "S": S, "us_per_launch": round(us, 2), "featurizes_per_s": n / us * 1e6,
                          "algorithmic_GBps": round(b / us / 1e3, 1), "frac_of_measured_hbm": round(b / us / 1e3 / PEAK, 4)}), flush=True)
    del env
    torch.cuda.empty_cache()
