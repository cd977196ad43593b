#!/usr/bin/env python
"""Config 5 (policy in the loop), kernel by kernel: a few EAGER transitions of selfplay.SelfPlayRollout so that
    ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file out.csv python tools/prof_selfplay.py
lists every launch of one transition; without ncu it prints CUDA-event times of the stages (encode / policy / sample / step)
and of the graph replay."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--eager", type=int, default=3, help="eager transitions (what ncu lists)")
ap.add_argument("--stages", action="store_true", help="time the stages with CUDA events")
ap.add_argument("--wide", type=int, default=1, help="K9 (the two wide layers as one wgmma kernel)")
ap.add_argument("--tail", type=int, default=1, help="K8 (dense tail + heads + draw in one kernel)")
ap.add_argument("--fused", type=int, default=1, help="K7 (encoding + first layer from the record) instead of K2 + first GEMM")
args = ap.parse_args()
env = BatchedOvercookedEnv(["cramped_room"], args.n, horizon=400, auto_reset=True)
sp = SelfPlayRollout(env, use_graph=False, fused_first_layer=bool(args.fused), fused_tail=bool(args.tail),
                     fused_wide=bool(args.wide and args.tail and args.fused))
for _ in range(args.eager):
    sp._transition()
torch.cuda.synchronize()
if args.stages:
    def ev():
        return torch.cuda.Event(enable_timing=True)

    def timed(fn, reps=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps * 1e3  # us

    N, W, H = env.n_envs, sp.W, sp.H
    out = {"n_envs": N}
    obs = sp.obs if sp.obs is not None else torch.empty((N, 2, W, H, 26), dtype=torch.bfloat16, device=env.device)
    out["fused_first_layer"] = sp.fused_first_layer
    out["encode_us"] = timed(lambda: env.lossless_state_encoding(out=obs))
    wt0, b0 = sp.dense_model.first_layer_table()
    act0 = torch.empty((2 * N, wt0.shape[1]), dtype=torch.bfloat16, device=env.device)
    out["k7_encode_linear_us"] = timed(lambda: env.encoded_linear(wt0, b0, out=act0, neg_slope=0.2))
    out["fused_tail"] = sp.fused_tail
    out["fused_wide"] = sp.fused_wide
    if sp.fused_wide:
        from overcooked_ai_b200 import _native as _nv
        w1_, b1_, w2_, b2_ = sp._wide
        a0_ = torch.randn((2 * N, 512), device=env.device).to(torch.bfloat16)
        z_ = torch.empty((2 * N, 160), dtype=torch.bfloat16, device=env.device)
        out["k9_wide_layers_us"] = timed(lambda: _nv.check(_nv.lib().ovc_wide_layers(a0_.data_ptr(), 2 * N, 512, w1_.data_ptr(), b1_.data_ptr(), 512,
                                                                                       w2_.data_ptr(), b2_.data_ptr(), 160, 0.2, z_.data_ptr(), env._stream())))
    out["policy_us"] = timed(sp._policy)
    from overcooked_ai_b200 import _native
    w1, b1, wh, bh, wo, bo = sp.dense_model.tail_tables()
    z = torch.randn((2 * N, w1.shape[1]), device=env.device).to(torch.bfloat16)
    vals = torch.empty(2 * N, dtype=torch.float32, device=env.device)
    out["k8_policy_tail_us"] = timed(lambda: _native.check(_native.lib().ovc_policy_tail(
        z.data_ptr(), 2 * N, z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0], wo.data_ptr(),
        bo.data_ptr(), 0.3, 6, 1, sp._draw_counter.data_ptr(), sp.actions.data_ptr(), vals.data_ptr(), 0, env._stream())))
    x = obs.view(2 * N, W * H * 26)
    with torch.no_grad():
        layers = list(sp.dense_model.conv_as_linear) + list(sp.dense_model.dense) + [sp.dense_model.heads]
        for i, lin in enumerate(layers):
            out["layer%d_%dx%d_linear_us" % (i, lin.in_features, lin.out_features)] = timed(lambda: lin(x))
            y = lin(x)
            if i < len(layers) - 1:
                out["layer%d_lrelu_us" % i] = timed(lambda: torch.nn.functional.leaky_relu(y, 0.2, inplace=True))
            x = y
    out["sample_us"] = timed(lambda: env.sample_actions(sp._scores, sp._draw_counter, seed=1, out=sp.actions))
    out["step_us"] = timed(lambda: env.step(sp.actions))
    out["record_transition_us"] = timed(lambda: env.record_transition(sp._factor, ret_sparse=sp.ret_sparse, ret_mixed=sp.ret_mixed))
    out["transition_eager_us"] = timed(sp._transition)
    spg = SelfPlayRollout(env, use_graph=True, fused_first_layer=sp.fused_first_layer, fused_tail=sp.fused_tail, fused_wide=sp.fused_wide)
    spg.run(4)
    out["transition_graph_us"] = timed(lambda: spg.run(1))
    print(json.dumps(out))
print("done")
