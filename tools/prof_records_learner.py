#!/usr/bin/env python
"""Cost of one PPO epoch on one collect(400) batch of cramped_room at 32 768 envs (13.1 M env-steps), at the loss of
examples/ppo_selfplay.py with Adam, written as one JSON file under --out:

  (a) K2 float32 observation + RllibShapedCNN (cuDNN convolutions): the example's default learner;
  (b) K2 bf16 observation + the folded GEMMs: SampleBatch.forward(..., fused_first_layer=False);
  (c) SampleBatch.forward: K7 on the records forward, K12 for the first layer's weight gradient;
  each path one epoch at a time, alternated (a b c a b c ...), timed with CUDA events, each on its own copy of the
  network and optimizer;
  K12 alone against the dense bf16 GEMM obs^T dz on K2's observation of the same rows (and K2 itself), with K12's
  achieved bytes/s from shape-computed traffic: dz once, the records once per column slice, the dwt flush (every CTA's
  whole slice: an upper bound, zero sums are skipped);
  max |ratio - 1| at the first minibatch (before any update) for (a) and (c);
  the card's name and power limit, read in the same run.

    python tools/prof_records_learner.py --out DIR
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--n", type=int, default=32768)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--minibatch-rows", type=int, default=65536, help="agent rows per minibatch (two per env-step)")
ap.add_argument("--rounds", type=int, default=2, help="epochs per path, alternated")
ap.add_argument("--reps", type=int, default=20, help="K12 / GEMM launches per timing")
args = ap.parse_args()
assert torch.cuda.is_available(), "prof_records_learner measures on a CUDA device"


def ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


N, T = args.n, args.steps
torch.manual_seed(0)
env = BatchedOvercookedEnv("cramped_room", N, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibShapedCNN(W, H).cuda()
sp = SelfPlayRollout(env, model=model, seed=0)
batch = sp.collect(T, 0.99, 0.98)
torch.cuda.synchronize()
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = {"gpu": gpu.splitlines()[0] if gpu else torch.cuda.get_device_name(), "n_envs": N, "steps": T, "layout": "cramped_room",
       "minibatch_rows": args.minibatch_rows, "env_steps": N * T}

adv_all = batch.advantages.view(-1)
adv_all = (adv_all - adv_all.mean()) / (adv_all.std() + 1e-8)
old_logp, targets, actions = batch.logp.view(-1), batch.value_targets.view(-1), batch.actions.view(-1).long()
mb = args.minibatch_rows // 2  # env-steps per minibatch


def loss_of(logits, value, rows, clip=0.05):
    logp_all = F.log_softmax(logits, dim=-1)
    ratio = torch.exp(logp_all.gather(1, actions[rows, None]).squeeze(1) - old_logp[rows])
    a = adv_all[rows]
    policy = -torch.min(ratio * a, ratio.clamp(1 - clip, 1 + clip) * a).mean()
    entropy = -(logp_all.exp() * logp_all).sum(-1).mean()
    return policy + 1e-4 * F.mse_loss(value, targets[rows]) - 0.1 * entropy, ratio


def fwd_a(m, idx):
    obs = batch.observations(idx).view(-1, W, H, 26).permute(0, 3, 1, 2)
    return m(obs)


paths = {"a_k2_f32_conv": fwd_a,
         "b_k2_bf16_folded": lambda m, idx: batch.forward(m, idx, fused_first_layer=False),
         "c_records_k7_k12": lambda m, idx: batch.forward(m, idx)}
state = {k: (copy.deepcopy(model), None) for k in paths}
state = {k: (m, torch.optim.Adam(m.parameters(), lr=1e-3)) for k, (m, _) in state.items()}

# first-minibatch ratio, before any update, on the same env-steps
g = torch.Generator(device="cuda")
g.manual_seed(1)
perm0 = torch.randperm(N * T, device="cuda", generator=g)
idx0 = perm0[:mb]
rows0 = (2 * idx0[:, None] + torch.arange(2, device="cuda")).view(-1)
for k in ("a_k2_f32_conv", "c_records_k7_k12", "b_k2_bf16_folded"):
    with torch.no_grad():
        _, ratio = loss_of(*paths[k](state[k][0], idx0), rows0)
    out["first_minibatch_max_abs_ratio_minus_1_" + k] = float((ratio - 1).abs().max())


def epoch(k, n_minibatches=None):
    m, opt = state[k]
    perm = torch.randperm(N * T, device="cuda")
    stop = N * T if n_minibatches is None else n_minibatches * mb
    for s in range(0, stop, mb):
        idx = perm[s:s + mb]
        rows = (2 * idx[:, None] + torch.arange(2, device="cuda")).view(-1)
        loss, _ = loss_of(*paths[k](m, idx), rows)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()


for k in paths:  # warm every shape the timed epochs use
    epoch(k, 3)
torch.cuda.synchronize()
times = {k: [] for k in paths}
for _ in range(args.rounds):
    for k in paths:
        times[k].append(ms(lambda: epoch(k)))
for k, v in times.items():
    out["epoch_ms_" + k] = v
out["minibatches_per_epoch"] = -(-N * T // mb)
out["epoch_b_over_c"] = min(times["b_k2_bf16_folded"]) / min(times["c_records_k7_k12"])
out["epoch_a_over_c"] = min(times["a_k2_f32_conv"]) / min(times["c_records_k7_k12"])

# K12 alone against the dense weight-gradient GEMM on K2's bf16 observation, at one minibatch's rows
idx = perm0[:mb]
recs = batch.states.view(-1, batch.states.shape[-1]).index_select(0, idx)
n_out = 512
dz = torch.randn((2 * mb, n_out), device="cuda")
dwt = torch.zeros((W * H * 26, n_out), device="cuda")
obs = env.lossless_state_encoding(dtype=torch.bfloat16, states=recs).view(2 * mb, -1)
dz16 = dz.to(torch.bfloat16)
runs = {"k12_wgrad": lambda: env.encoded_linear_wgrad(recs, dz, dwt),
        "k2_bf16_encode": lambda: env.lossless_state_encoding(dtype=torch.bfloat16, states=recs),
        "gemm_obsT_dz_bf16": lambda: torch.mm(obs.t(), dz16)}
for f in runs.values():
    f()
torch.cuda.synchronize()
for _ in range(3):
    for k, f in runs.items():
        out.setdefault(k + "_us", []).append(ms(lambda: [f() for _ in range(args.reps)]) * 1e3 / args.reps)
props = torch.cuda.get_device_properties(0)
n_sm = props.multi_processor_count
cs = 128  # K12's column slice at 5x4 (4 columns per lane)
n_slices = n_out // cs
workers = max(1, n_sm // n_slices)
traffic = {"dz": 2 * mb * n_out * 4, "records": mb * env.state_words * 4 * n_slices,
           "dwt_flush": workers * n_slices * W * H * 19 * cs * 4}
out["k12_traffic_bytes"] = traffic
out["k12_gb_per_s"] = sum(traffic.values()) / (min(out["k12_wgrad_us"]) * 1e-6) / 1e9
out["gemm_gflop"] = 2.0 * 2 * mb * W * H * 26 * n_out / 1e9

os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "prof_records_learner.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print(json.dumps(out))
print("wrote", path)
