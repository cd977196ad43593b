#!/usr/bin/env python
"""Fictitious co-play's first stage: K independent PPO self-play agents from different seeds, trained in ONE device rollout,
their checkpoints saved as the population of the second stage.

``SelfPlayRollout(env, [m_0, ..., m_{K-1}])`` gives member k the environments of its block ``[o_k, o_{k+1})``; one
``collect()`` returns the ordinary two-view ``SampleBatch``, whose joint rows ``[2 o_k, 2 o_{k+1})`` are member k's.  Each
member has its own Adam optimizer and trains only on its block's env-steps ``t * N + e`` through ``batch.forward`` (the
folded bf16 network the rollout runs, evaluated from the stored records), with the clipped PPO objective.  After each
iteration ``sync_weights()`` refolds every member; the captured CUDA graph keeps running.  At the end each member's state
dict is written to ``--save-dir/member_k.pt``, which ``examples/ppo_population.py --members`` loads (stage 2).  A
demonstration, not library code: no entropy schedule, no KL penalty, one process.

    python examples/ppo_selfplay_population.py --k 4 --iters 5 --save-dir /tmp/fcp
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--k", type=int, default=4, help="population members (independent self-play agents)")
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=4096)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=4096, help="env-steps per minibatch of one member")
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--gamma", type=float, default=0.99)
ap.add_argument("--lam", type=float, default=0.98)
ap.add_argument("--clip", type=float, default=0.05)
ap.add_argument("--vf-coef", type=float, default=1e-4)
ap.add_argument("--entropy-coef", type=float, default=0.1)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--save-dir", default=None, help="write member_k.pt state dicts here")
args = ap.parse_args()

env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
members = []
for k in range(args.k):  # a different initialisation per member
    torch.manual_seed(args.seed * 1000 + k)
    members.append(RllibShapedCNN(W, H).cuda())
sp = SelfPlayRollout(env, model=members, seed=args.seed)
opts = [torch.optim.Adam(m.parameters(), lr=args.lr) for m in members]
offs = sp.blocks.tolist()
N, T = env.n_envs, args.steps
steps = torch.arange(T, device=env.device)[:, None] * N
for it in range(args.iters):
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    member_of_episode = sp.member[fin["env_index"]]
    line = []
    for k, (m, opt) in enumerate(zip(members, opts)):
        a, b = offs[k], offs[k + 1]
        env_steps = (steps + torch.arange(a, b, device=env.device)[None, :]).reshape(-1)  # member k's env-steps t * N + e
        rows = torch.stack([2 * env_steps, 2 * env_steps + 1], 1).reshape(-1)  # both agent rows of each, in forward()'s order
        adv = batch.advantages.view(-1)[rows]
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
        old_logp, targets = batch.logp.view(-1)[rows], batch.value_targets.view(-1)[rows]
        actions = batch.actions.view(-1)[rows].long()
        for epoch in range(args.epochs):
            perm = torch.randperm(env_steps.numel(), device=env.device)
            for i in range(0, env_steps.numel(), args.minibatch):
                mb = perm[i:i + args.minibatch]
                r = torch.stack([2 * mb, 2 * mb + 1], 1).reshape(-1)
                logits, values = batch.forward(m, env_steps[mb])
                logp_all = F.log_softmax(logits, -1)
                ratio = torch.exp(logp_all.gather(1, actions[r, None]).squeeze(1) - old_logp[r])
                pg = -torch.min(ratio * adv[r], ratio.clamp(1 - args.clip, 1 + args.clip) * adv[r]).mean()
                vf = F.mse_loss(values, targets[r])
                ent = -(logp_all.exp() * logp_all).sum(-1).mean()
                loss = pg + args.vf_coef * vf - args.entropy_coef * ent
                opt.zero_grad()
                loss.backward()
                opt.step()
        sel = member_of_episode == k
        line.append("m%d %.2f" % (k, float(fin["ep_sparse_r"][sel].float().mean()) if bool(sel.any()) else float("nan")))
    sp.sync_weights()
    print("iter %d  collect %.1f ms  mean sparse return per member: %s" % (it, t_collect * 1e3, "  ".join(line)), flush=True)
if args.save_dir:
    os.makedirs(args.save_dir, exist_ok=True)
    for k, m in enumerate(members):
        torch.save(m.state_dict(), os.path.join(args.save_dir, "member_%d.pt" % k))
    print("saved %d members to %s (examples/ppo_population.py --members %s/member_*.pt)" % (args.k, args.save_dir, args.save_dir))
