"""The reference's own Python path timed on this host's cores (SURVEY.md §8d "CPU baseline beside it", items 1-3):
OvercookedEnv.step and lossless_state_encoding_mdp, one process, then one process per visible core.
TEST / MEASUREMENT INFRASTRUCTURE: imports the unmodified reference through oracle/refboot.py (OVC_REFERENCE or the
oracle/_ref copy); bench.py's reference arm times the C port, which needs no reference checkout.

    python tools/ref_python_baseline.py [episodes]
"""
import multiprocessing as mp
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
LAYOUTS = ["cramped_room", "asymmetric_advantages", "coordination_ring", "forced_coordination", "counter_circuit"]


def run(args):
    layout, episodes, seed, encode = args
    from oracle import refboot

    ns = refboot.boot()
    m = refboot.make_mdp(ns, layout)
    env = refboot.make_env(ns, m, horizon=400)
    env._mp = object()  # the planner is not on the step path; never let it be computed / pickled (SURVEY appendix E)
    rng = np.random.RandomState(seed)
    acts = [ns.actions.Action.INDEX_TO_ACTION[i] for i in range(6)]
    n = 0
    t0 = time.perf_counter()
    for _ in range(episodes):
        env.reset(regen_mdp=False)
        done = False
        while not done:
            a = rng.randint(0, 6, size=2)
            state, _, done, _ = env.step((acts[a[0]], acts[a[1]]))
            if encode:
                env.lossless_state_encoding_mdp(state)
            n += 1
    return n, time.perf_counter() - t0


def main():
    episodes = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    print("reference Python path, build container, %d logical cores visible, %d episodes x 400 steps per layout" % (os.cpu_count(), episodes))
    print("| layout | step only, 1 process (steps/s) | step + lossless encoding, 1 process (steps/s) |")
    print("|---|---|---|")
    for layout in LAYOUTS:
        n, dt = run((layout, episodes, 0, False))
        n2, dt2 = run((layout, max(2, episodes // 4), 0, True))
        print("| %s | %.0f | %.0f |" % (layout, n / dt, n2 / dt2))
    procs = os.cpu_count() or 1
    with mp.get_context("fork").Pool(procs) as pool:
        t0 = time.perf_counter()
        res = pool.map(run, [("cramped_room", episodes, k, False) for k in range(procs)])
        wall = time.perf_counter() - t0
    print("\ncramped_room, %d processes (one env each): %.0f steps/s aggregate (wall %.1f s; per-process %.0f .. %.0f)"
          % (procs, sum(r[0] for r in res) / wall, wall, min(r[0] / r[1] for r in res), max(r[0] / r[1] for r in res)))


if __name__ == "__main__":
    main()
