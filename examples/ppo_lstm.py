#!/usr/bin/env python
"""PPO self-play with the reference's LSTM model (``use_lstm``) on cramped_room: this library as the rollout worker, a
plain torch learner with backpropagation through time.

The worker (``SelfPlayRollout.collect`` with ``RllibLSTMShapedCNN``) runs K7 -> K9 -> K8's hidden output -> K11 (the LSTM
cell, the heads and the draw) and the environments on the GPU.  Its ``SampleBatch`` cuts the window into chunks of
``max_seq_len`` transitions and holds the state each chunk started from (``state_h`` / ``state_c``).  The learner draws
minibatches of (chunk, environment) sequences, starts each from that state, runs ``forward_sequence`` over the
re-encoded observations with the state zeroed after every ``dones[t - 1]``, and uses the clipped PPO objective of
``examples/ppo_selfplay.py``.  ``sync_weights()`` folds the update back into the kernels' tables.

The first minibatch's max |ratio - 1| is printed: it is small only if the learner's sequences start from the state the
worker used and follow the same resets (besides the bf16 fold of the weights, as in ``ppo_selfplay.py``).  A
demonstration, not library code.

    python examples/ppo_lstm.py --iters 5
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import RllibLSTMShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=1024)
ap.add_argument("--steps", type=int, default=400, help="transitions per window (one episode at horizon 400)")
ap.add_argument("--max-seq-len", type=int, default=20, help="RLlib's max_seq_len: transitions per sequence")
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=512, help="(chunk, environment) sequences per minibatch")
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--gamma", type=float, default=0.99)
ap.add_argument("--lam", type=float, default=0.98)
ap.add_argument("--clip", type=float, default=0.05)
ap.add_argument("--vf-coef", type=float, default=1e-4)
ap.add_argument("--entropy-coef", type=float, default=0.1)
ap.add_argument("--seed", type=int, default=0)
args = ap.parse_args()

torch.manual_seed(args.seed)
env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibLSTMShapedCNN(W, H).cuda()
sp = SelfPlayRollout(env, model=model, seed=args.seed, max_seq_len=args.max_seq_len)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T, L = env.n_envs, args.steps, args.max_seq_len
assert T % L == 0, "whole sequences only in this example"
K = T // L
dev = env.device
agents = torch.arange(2, device=dev)
for it in range(args.iters):
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    episodes = fin["env_index"].numel()
    mean_sparse = float(fin["ep_sparse_r"].float().mean()) if episodes else float("nan")
    adv = batch.advantages
    adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    # reset[t] = dones[t - 1] within a chunk (the state at t = k L is stored after the rule already)
    reset_all = torch.zeros((T, N), dtype=torch.uint8, device=dev)
    reset_all[1:] = batch.dones[:-1]
    reset_all[::L] = 0
    first_ratio = None
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(K * N, device=dev)
        for m in range(0, K * N, args.minibatch):
            seq = perm[m:m + args.minibatch]
            k, e = seq // N, seq % N
            M = seq.numel()
            t_idx = k[None, :] * L + torch.arange(L, device=dev)[:, None]            # [L, M]
            rows = (2 * e[:, None] + agents).view(-1)                                   # [2M] agent rows of the sequences
            obs = batch.observations((t_idx * N + e[None, :]).view(-1))                 # [L M, 2, W, H, 26]
            obs = obs.view(L, 2 * M, W, H, 26).permute(0, 1, 4, 2, 3)
            reset = reset_all[t_idx, e[None, :]].repeat_interleave(2, 1)                # [L, 2M]
            h0 = batch.state_h[k[:, None], rows.view(M, 2)].view(2 * M, -1).float()
            c0 = batch.state_c[k[:, None], rows.view(M, 2)].view(2 * M, -1)
            logits, value, _ = model.forward_sequence(obs, h0, c0, reset)              # [L, 2M, 6], [L, 2M]
            act = batch.actions[t_idx[:, :, None], rows.view(M, 2)[None]].view(L, 2 * M).long()
            old_logp = batch.logp[t_idx[:, :, None], rows.view(M, 2)[None]].view(L, 2 * M)
            a = adv[t_idx[:, :, None], rows.view(M, 2)[None]].view(L, 2 * M)
            targets = batch.value_targets[t_idx[:, :, None], rows.view(M, 2)[None]].view(L, 2 * M)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(2, act[..., None]).squeeze(2)
            ratio = torch.exp(logp - old_logp)
            if first_ratio is None:
                first_ratio = float((ratio.detach() - 1).abs().max())
            policy_loss = -torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a).mean()
            value_loss = F.mse_loss(value, targets)
            entropy = -(logp_all.exp() * logp_all).sum(-1).mean()
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    sp.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  episodes %d  mean sparse return %.2f  first-minibatch max|ratio-1| %.4f  policy loss %.4f  value loss %.3f  "
          "entropy %.3f  collect %.2f s  learn %.2f s"
          % (it, episodes, mean_sparse, first_ratio, policy_loss.item(), value_loss.item(), entropy.item(), t_collect,
             time.time() - t0), flush=True)
