#!/usr/bin/env python
"""PPO against a frozen partner on cramped_room: a best response to a fixed agent, or the second stage of a population
method such as fictitious co-play (the learner trains next to frozen checkpoints), with this library as the rollout worker.

``AgentPairRollout((learner, partner), random_seats=True).collect()`` runs the learner's policy on its own seat only
(one-view K7 -> K9 -> K8), the partner on the other seat, the environments (K1), the learner's reward and the seat draw:
every episode starts with the players drawn again, as the reference's gym wrapper does at every reset.  The batch holds
one row per environment, the learner's, so the loss needs no mask.  The partner never changes; after each update
``pair.sync_weights()`` folds the learner's new weights into the captured graph.  To train against a population with a
member drawn per episode, see ``examples/ppo_population.py``.

The partner is a randomly initialised ``RllibShapedCNN`` unless ``--partner`` names a ``torch.save``d state dict of one, or
``--bc`` makes it a (randomly initialised) ``BCPolicy``.  A demonstration, not library code.

    python examples/ppo_partner.py --iters 5
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
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=8192, help="env-steps per minibatch (one learner row each)")
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--gamma", type=float, default=0.99)
ap.add_argument("--lam", type=float, default=0.98)
ap.add_argument("--clip", type=float, default=0.05)
ap.add_argument("--vf-coef", type=float, default=1e-4)
ap.add_argument("--entropy-coef", type=float, default=0.1)
ap.add_argument("--shaping-horizon", type=float, default=2.5e6, help="env-steps over which the shaping factor anneals 1 -> 0")
ap.add_argument("--partner", default=None, help="state dict of an RllibShapedCNN checkpoint (default: random init)")
ap.add_argument("--bc", action="store_true", help="a BCPolicy partner instead of a PPO network")
ap.add_argument("--bootstrap-horizon", action="store_true",
                help="bootstrap the advantages from the value of each episode's last state at the horizon cut")
ap.add_argument("--seed", type=int, default=0)
args = ap.parse_args()

torch.manual_seed(args.seed)
env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibShapedCNN(W, H).cuda()
partner = BCPolicy() if args.bc else RllibShapedCNN(W, H)
if args.partner:
    partner.load_state_dict(torch.load(args.partner, map_location="cpu"))
pair = AgentPairRollout(env, (model, partner), seed=args.seed, random_seats=True)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
env_steps = 0
for it in range(args.iters):
    pair.reward_shaping_factor = max(0.0, 1.0 - env_steps / args.shaping_horizon)
    t0 = time.time()
    batch = pair.collect(T, args.gamma, args.lam, bootstrap_horizon=args.bootstrap_horizon)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    episodes = fin["env_index"].numel()
    mean_return = float(fin["ep_sparse_r"].float().mean()) if episodes else float("nan")
    env_steps += T * N
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
    pair.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  shaping %.3f  learner in seat 0 %.3f  episodes %d  mean sparse return %.2f  policy loss %.4f  value loss %.3f  "
          "entropy %.3f  collect %.2f s  learn %.2f s"
          % (it, pair.reward_shaping_factor, float((batch.partner_seat == 1).float().mean()), episodes, mean_return,
             policy_loss.item(), value_loss.item(), entropy.item(), t_collect, time.time() - t0), flush=True)
