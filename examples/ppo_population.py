#!/usr/bin/env python
"""Fictitious co-play's second stage on cramped_room: PPO against a population of K frozen checkpoints, one drawn per
episode, with this library as the rollout worker.

``AgentPairRollout((learner, [m_0, ..., m_K-1]), random_seats=True)`` draws each environment's member at construction and
again at every episode end (``member_weights``, uniform by default), and runs each member's policy on its own environments
only.  Every PPO batch therefore mixes all members across the environments, instead of playing one member per window.
``episodes.finished()["partner_member"]`` says which member each finished episode was played with, so the script prints the
mean return per member: one row of the cross-play matrix per window.  Setting ``pop.member_weights`` between windows
(e.g. towards the members the learner does worst against) takes effect without a re-capture.

The members are randomly initialised ``RllibShapedCNN``s unless ``--members`` names ``torch.save``d state dicts of them;
``--bc K`` adds K (randomly initialised) ``BCPolicy`` members.  A demonstration, not library code.

    python examples/ppo_population.py --iters 5 --k 4
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=2048)
ap.add_argument("--steps", type=int, default=400, help="transitions per window (one episode at horizon 400)")
ap.add_argument("--k", type=int, default=4, help="randomly initialised PPO members (without --members)")
ap.add_argument("--members", nargs="*", default=None, help="state dicts of RllibShapedCNN checkpoints, one per member")
ap.add_argument("--bc", type=int, default=0, help="BCPolicy members added to the population")
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=8192, help="env-steps per minibatch (one learner row each)")
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
model = RllibShapedCNN(W, H).cuda()
members = []
for path in args.members or [None] * args.k:
    m = RllibShapedCNN(W, H)
    if path:
        m.load_state_dict(torch.load(path, map_location="cpu"))
    members.append(m)
members += [BCPolicy() for _ in range(args.bc)]
K = len(members)
pop = AgentPairRollout(env, (model, members), seed=args.seed, random_seats=True, episode_capacity=1)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
for it in range(args.iters):
    t0 = time.time()
    batch = pop.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    ret, mem = fin["ep_sparse_r"].float(), fin["partner_member"].long()
    per_member = torch.zeros(K, device=env.device).index_add_(0, mem, ret)
    count = torch.bincount(mem, minlength=K).float()
    adv = batch.advantages.view(-1)
    adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    old_logp, targets, actions = batch.logp.view(-1), batch.value_targets.view(-1), batch.actions.view(-1).long()
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(T * N, device=env.device)
        for k in range(0, T * N, args.minibatch):
            idx = perm[k:k + args.minibatch]
            obs = batch.observations(idx).permute(0, 3, 1, 2)  # the learner's own view, [M, 26, W, H]
            logits, value = model(obs)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(1, actions[idx, None]).squeeze(1)
            ratio = torch.exp(logp - old_logp[idx])
            a = adv[idx]
            policy_loss = -torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a).mean()
            value_loss = ((value - targets[idx]) ** 2).mean()
            entropy = (-(logp_all.exp() * logp_all).sum(-1)).mean()
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    pop.sync_weights()
    torch.cuda.synchronize()
    means = (per_member / count.clamp(min=1)).tolist()
    print("iter %d  episodes %d  mean sparse return per member [%s]  policy loss %.4f  collect %.2f s  learn %.2f s"
          % (it, int(count.sum()), ", ".join("%d: %.2f (%d)" % (k, r, c) for k, (r, c) in enumerate(zip(means, count.long().tolist()))),
             policy_loss.item(), t_collect, time.time() - t0), flush=True)
