#!/usr/bin/env python
"""Quick GPU sanity check of one record-I/O strategy of the step kernel against the CPU oracle.
Run under `timeout` on the GPU before the full test-suite:  python tools/gpu_sanity.py --io 1"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

from oracle import cpu  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--io", type=int, default=1)
ap.add_argument("--n", type=int, default=1000)
ap.add_argument("--layouts", default="cramped_room")
args = ap.parse_args()
layouts = args.layouts.split(",")
print("device", torch.cuda.get_device_name(0), "io", args.io, "layouts", layouts, flush=True)
env = BatchedOvercookedEnv(layouts, args.n, horizon=50, io=args.io, auto_reset=True)
rng = np.random.RandomState(0)
T = 60
acts = rng.randint(0, 6, size=(T, args.n, 2)).astype(np.int32)
acts[rng.rand(T, args.n, 2) < 0.3] = 5
ref_state = env.state.cpu().numpy().copy()
ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=50, flags=1, n_threads=2)
d = torch.from_numpy(acts).cuda()
t0 = time.time()
for t in range(T // 2):
    out = env.step(d[t])
    torch.cuda.synchronize()
    for name, got, want in zip(("sparse", "shaped", "done", "events"), out, ref):
        if not np.array_equal(got.cpu().numpy(), want[t]):
            bad = np.nonzero((got.cpu().numpy() != want[t]).reshape(args.n, -1).any(1))[0]
            print("FAIL step t=%d %s, %d envs differ, first %s" % (t, name, len(bad), bad[:5]))
            sys.exit(1)
out = env.rollout(d[T // 2:].contiguous())
torch.cuda.synchronize()
for name, got, want in zip(("sparse", "shaped", "done", "events"), out, ref):
    if not np.array_equal(got.cpu().numpy(), want[T // 2:]):
        print("FAIL rollout", name)
        sys.exit(1)
if not np.array_equal(env.state.cpu().numpy(), ref_state):
    print("FAIL final state")
    sys.exit(1)
print("OK io=%d S=%d in %.2fs" % (args.io, env.state_words, time.time() - t0))
