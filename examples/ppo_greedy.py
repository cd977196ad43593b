#!/usr/bin/env python
"""PPO next to the reference's scripted GreedyHumanModel on cramped_room: a best response to the standard human-like
baseline partner, with nothing trained beforehand (no PPO checkpoint, no BC weights), with this library as the rollout
worker.

``AgentPairRollout((learner, GreedyHumanModel()), random_seats=True).collect()`` runs the learner's policy on its own seat
(one-view K7 -> K9 -> K8), the greedy agent on the other seat (``ovc_greedy_actions``: the reference's goal choice over
per-layout motion-plan tables, one thread per environment), the environments (K1), the learner's reward and the seat draw.
The batch holds one row per environment, the learner's.  ``--bc-factor`` below 1 instead trains with
``SelfPlayRollout(partner=GreedyHumanModel(), bc_factor=...)``: each episode is self-play or played next to the greedy
agent, and the loss is averaged over ``batch.learner_mask``.  A demonstration, not library code.

    python examples/ppo_greedy.py --iters 5
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.greedy import GreedyHumanModel  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN, SelfPlayRollout  # noqa: E402

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
ap.add_argument("--bc-factor", type=float, default=1.0, help="share of episodes played next to the greedy agent")
ap.add_argument("--seed", type=int, default=0)
args = ap.parse_args()

torch.manual_seed(args.seed)
env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibShapedCNN(W, H).cuda()
if args.bc_factor >= 1.0:
    pair = AgentPairRollout(env, (model, GreedyHumanModel()), seed=args.seed, random_seats=True)
else:
    pair = SelfPlayRollout(env, model=model, seed=args.seed, partner=GreedyHumanModel(), bc_factor=args.bc_factor)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
env_steps = 0
for it in range(args.iters):
    pair.reward_shaping_factor = max(0.0, 1.0 - env_steps / args.shaping_horizon)
    t0 = time.time()
    batch = pair.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    fin = batch.episodes.finished()
    episodes = fin["env_index"].numel()
    mean_return = float(fin["ep_sparse_r"].float().mean()) if episodes else float("nan")
    env_steps += T * N
    # one learner row per environment next to the pair; both rows, masked to the learner's, in a self-play mixture
    mask = batch.learner_mask.reshape(T * N, -1).float()
    views = mask.shape[1]
    adv = batch.advantages.reshape(T * N, views)
    mean = (adv * mask).sum() / mask.sum()
    adv = (adv - mean) / ((((adv - mean) ** 2 * mask).sum() / mask.sum()).sqrt() + 1e-8)
    old_logp, targets = batch.logp.reshape(T * N, views), batch.value_targets.reshape(T * N, views)
    actions = batch.actions.reshape(T * N, views).long()
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(T * N, device=env.device)
        for k in range(0, T * N, args.minibatch):
            idx = perm[k:k + args.minibatch]
            m = mask[idx].view(-1)
            obs = batch.observations(idx).reshape(-1, W, H, 26).permute(0, 3, 1, 2)  # [M * views, 26, W, H]
            logits, value = model(obs)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(1, actions[idx].view(-1, 1)).squeeze(1)
            ratio = torch.exp(logp - old_logp[idx].view(-1))
            a = adv[idx].view(-1)
            masked_mean = lambda x: (x * m).sum() / m.sum().clamp(min=1)  # noqa: E731  the learner's rows only
            policy_loss = -masked_mean(torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a))
            value_loss = masked_mean((value - targets[idx].view(-1)) ** 2)
            entropy = masked_mean(-(logp_all.exp() * logp_all).sum(-1))
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    pair.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  shaping %.3f  paired env-steps %.3f  episodes %d  mean sparse return %.2f  policy loss %.4f  value loss %.3f  "
          "entropy %.3f  collect %.2f s  learn %.2f s"
          % (it, pair.reward_shaping_factor, float((batch.partner_seat >= 0).float().mean()), episodes, mean_return,
             policy_loss.item(), value_loss.item(), entropy.item(), t_collect, time.time() - t0), flush=True)
