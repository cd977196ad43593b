#!/usr/bin/env python
"""The reference's OWN Python step timed on this machine's host cores (SURVEY.md §8(d) "CPU baseline beside it"):
the unmodified OvercookedEnv.step loop (reference overcooked_env.py:244-274, reset :288-319) under uniform random
joint actions, horizon 400 — (1) one process pinned to one core, (2) one process per usable core, all pinned,
started together behind a barrier; optionally (3) the same with lossless_state_encoding_mdp after every step.

TEST / MEASUREMENT INFRASTRUCTURE: imports the reference through oracle/refboot.py (OVC_REFERENCE, or
the oracle/_ref copy).  Runs in its own process (bench.py spawns it: no CUDA context is ever
forked).  Prints ONE JSON line.

    python oracle/ref_python_bench.py [--layout cramped_room] [--seconds 4] [--encode]
"""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def usable_cpus():
    """CPUs this process may run on: the affinity mask capped by the cgroup quota."""
    cpus = sorted(os.sched_getaffinity(0))
    lim = 0
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            lim = -(-int(q) // int(p))
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0 and p > 0:
                lim = -(-q // p)
        except Exception:
            pass
    return cpus[:lim] if 0 < lim < len(cpus) else cpus


def worker(cpu, layout, seconds, encode, seed, barrier, q):
    try:
        os.sched_setaffinity(0, {cpu})
    except Exception:
        pass
    from oracle import refboot

    ns = refboot.boot()
    m = refboot.make_mdp(ns, layout)
    env = refboot.make_env(ns, m, horizon=400)  # env._mp sentinel: the planner is not on the step path (SURVEY 8c hazard)
    acts = [ns.actions.Action.INDEX_TO_ACTION[i] for i in range(6)]
    trace = np.random.RandomState(seed).randint(0, 6, size=(64, 400, 2))
    for a in trace[0][:50]:  # warm the interpreter's caches
        env.step((acts[a[0]], acts[a[1]]))
    if barrier is not None:
        barrier.wait()
    n, ep = 0, 0
    t0 = time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        env.reset(regen_mdp=False)
        for a in trace[ep % 64]:
            state, _, done, _ = env.step((acts[a[0]], acts[a[1]]))
            if encode:
                env.lossless_state_encoding_mdp(state)
        assert done
        n, ep = n + 400, ep + 1
    q.put((n, time.perf_counter() - t0))


def run(cpus, layout, seconds, encode):
    ctx = mp.get_context("fork")
    q = ctx.Queue()
    barrier = ctx.Barrier(len(cpus)) if len(cpus) > 1 else None
    ps = [ctx.Process(target=worker, args=(c, layout, seconds, encode, k, barrier, q)) for k, c in enumerate(cpus)]
    for p in ps:
        p.start()
    res = [q.get() for _ in ps]
    for p in ps:
        p.join()
    # whole episodes only, so workers overrun `seconds` by up to one episode: aggregate = sum of per-process rates
    return sum(n / dt for n, dt in res), [n / dt for n, dt in res]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layout", default="cramped_room")
    ap.add_argument("--seconds", type=float, default=4.0)
    ap.add_argument("--encode", action="store_true")
    args = ap.parse_args()
    from oracle import refboot

    if not refboot.available():  # the workers would die in boot() and leave run() waiting for their results
        sys.exit("reference tree not found at %s" % refboot.REFERENCE_ROOT)
    cpus = usable_cpus()
    one, _ = run(cpus[:1], args.layout, args.seconds, False)
    allc, per = run(cpus, args.layout, args.seconds, False)
    out = {"what": "reference OvercookedEnv.step loop (overcooked_env.py:244-274), uniform random joint actions, horizon 400, whole episodes",
           "layout": args.layout, "source": refboot.REFERENCE_ROOT, "cores": len(cpus), "logical_cpus_online": os.cpu_count(),
           "steps_per_s_1core": one, "steps_per_s_all_cores": allc,
           "per_process_min_max": [min(per), max(per)], "seconds_per_leg": args.seconds}
    if args.encode:
        enc, _ = run(cpus, args.layout, args.seconds, True)
        out["steps_per_s_all_cores_with_lossless_encoding"] = enc
    print(json.dumps(out))


if __name__ == "__main__":
    main()
