#!/usr/bin/env python
"""PPO with a self-play mixture on cramped_room: each episode is self-play with probability ``1 - bc_factor`` and is played
next to a frozen PPO checkpoint otherwise, with the partner share annealed from 0 to 1 over the run (PPO_BC's
``bc_schedule`` with a network partner), and this library as the rollout worker.

``SelfPlayRollout(env, model, partner=frozen, bc_factor=f)`` draws each episode's seats at its start; the learner's policy
runs on its own rows only, and the partner on the seat it holds.  The batch keeps both rows of every environment;
``learner_mask`` drops the partner's rows from the loss.  The script prints the mean return of the finished episodes per
``partner_seat`` (-1: self-play); ``--members`` turns the partner into a population of frozen checkpoints and prints the
mean return per member as well.  A demonstration, not library code.

    python examples/ppo_mixture.py --iters 5
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
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=2048)
ap.add_argument("--steps", type=int, default=400, help="transitions per window (one episode at horizon 400)")
ap.add_argument("--members", type=int, default=0, help="a population of this many frozen checkpoints instead of one")
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=4096, help="env-steps per minibatch (both rows of each)")
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
frozen = [RllibShapedCNN(W, H) for _ in range(max(args.members, 1))]  # stand-ins for saved checkpoints
partner = frozen if args.members else frozen[0]
sp = SelfPlayRollout(env, model, partner=partner, bc_factor=0.0, seed=args.seed)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
for it in range(args.iters):
    sp.bc_factor = it / max(args.iters - 1, 1)  # the partner share, annealed 0 -> 1: a device scalar, no re-capture
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    ret, seat = fin["ep_sparse_r"].float(), fin["partner_seat"].long()
    report = ["seat %d: %.2f (%d)" % (s, ret[seat == s].mean().item(), int((seat == s).sum())) for s in (-1, 0, 1) if (seat == s).any()]
    if args.members:
        mem = fin["partner_member"].long()
        report += ["member %d: %.2f" % (k, ret[(seat >= 0) & (mem == k)].mean().item()) for k in range(args.members)
                   if ((seat >= 0) & (mem == k)).any()]
    mask = batch.learner_mask.view(T * N, 2).float()
    adv = batch.advantages.view(T * N, 2)
    sel = adv[mask.bool()]
    adv = (adv - sel.mean()) / (sel.std() + 1e-8)
    old_logp, targets = batch.logp.view(T * N, 2), batch.value_targets.view(T * N, 2)
    actions = batch.actions.view(T * N, 2).long()
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(T * N, device=env.device)
        for k in range(0, T * N, args.minibatch):
            idx = perm[k:k + args.minibatch]
            obs = batch.observations(idx).flatten(0, 1).permute(0, 3, 1, 2)  # both views, [2M, 26, W, H]
            logits, value = model(obs)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(1, actions[idx].view(-1, 1)).squeeze(1)
            m = mask[idx].view(-1)
            ratio = torch.exp(logp - old_logp[idx].view(-1))
            a = adv[idx].view(-1)
            denom = m.sum().clamp(min=1)
            policy_loss = -(torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a) * m).sum() / denom
            value_loss = (((value - targets[idx].view(-1)) ** 2) * m).sum() / denom
            entropy = ((-(logp_all.exp() * logp_all).sum(-1)) * m).sum() / denom
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    sp.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  bc_factor %.2f  mean sparse return [%s]  policy loss %.4f  collect %.2f s  learn %.2f s"
          % (it, sp.bc_factor, ", ".join(report), policy_loss.item(), t_collect, time.time() - t0), flush=True)
