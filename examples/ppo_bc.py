#!/usr/bin/env python
"""PPO_BC on cramped_room: PPO trained next to a fixed behaviour-cloned partner, the reference's human-proxy setup
(human_aware_rl's OvercookedMultiAgent with bc_factor / bc_schedule), with this library as the rollout worker.

Per transition the worker runs the PPO policy (K7 -> K9 -> K8) on both seats, then K10 overwrites the BC partner's seat
in the environments paired with it (featurize_state + the BC MLP + the draw, one kernel), then the environments (K1).  At
every episode start an environment is paired with the partner with probability ``bc_factor``, in a random seat.  The
learner is ``examples/ppo_selfplay.py``'s, with the loss averaged over ``batch.learner_mask`` so that the partner's
rows never train the PPO network.  ``bc_factor`` follows a piecewise-linear schedule of env-steps, as ``bc_schedule``
does, read by the captured graph without a re-capture.

The partner is a randomly initialised ``BCPolicy`` unless ``--bc-weights`` names an ``.npz`` with the reference's Keras
arrays ``dense_<i>_kernel`` / ``dense_<i>_bias`` and ``logits_kernel`` / ``logits_bias``.  A demonstration, not library
code.

    python examples/ppo_bc.py --iters 5
"""
import argparse
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import BCPolicy, RllibShapedCNN, SelfPlayRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=2048)
ap.add_argument("--steps", type=int, default=400, help="transitions per window (one episode at horizon 400)")
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=8192, help="env-steps per minibatch (two agent rows each)")
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--gamma", type=float, default=0.99)
ap.add_argument("--lam", type=float, default=0.98)
ap.add_argument("--clip", type=float, default=0.05)
ap.add_argument("--vf-coef", type=float, default=1e-4)
ap.add_argument("--entropy-coef", type=float, default=0.1)
ap.add_argument("--shaping-horizon", type=float, default=2.5e6, help="env-steps over which the shaping factor anneals 1 -> 0")
ap.add_argument("--bc-schedule", default="0:0,2e6:1", help="piecewise-linear bc_factor: env_steps:factor points, constant past the last")
ap.add_argument("--bc-weights", default=None, help=".npz of the BC model's Keras weights (default: random init)")
ap.add_argument("--seed", type=int, default=0)
args = ap.parse_args()


def schedule(points, x):
    """bc_schedule: linear between (env_steps, factor) points, constant outside them."""
    xs, ys = zip(*points)
    return float(np.interp(x, xs, ys))


points = sorted((float(a), float(b)) for a, b in (p.split(":") for p in args.bc_schedule.split(",")))
torch.manual_seed(args.seed)
env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibShapedCNN(W, H).cuda()
bc = BCPolicy()
if args.bc_weights:
    z = np.load(args.bc_weights)
    n_dense = len([k for k in z.files if k.startswith("dense_") and k.endswith("_kernel")])
    bc = BCPolicy(num_hidden_layers=n_dense).load_keras_weights(
        [(z["dense_%d_kernel" % i], z["dense_%d_bias" % i]) for i in range(n_dense)], (z["logits_kernel"], z["logits_bias"]))
sp = SelfPlayRollout(env, model=model, seed=args.seed, partner=bc, bc_factor=schedule(points, 0))
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
env_steps = 0
for it in range(args.iters):
    sp.reward_shaping_factor = max(0.0, 1.0 - env_steps / args.shaping_horizon)
    sp.bc_factor = schedule(points, env_steps)
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    paired = float((batch.partner_seat >= 0).float().mean())
    # the episodes that ended in the window, split by whether the BC partner played them
    fin = batch.episodes.finished()
    with_bc = fin["partner_seat"] >= 0
    episodes = fin["env_index"].numel()
    mean_return = lambda m: float(fin["ep_sparse_r"][m].float().mean()) if bool(m.any()) else float("nan")  # noqa: E731
    env_steps += T * N
    mask = batch.learner_mask.view(-1).float()
    adv = batch.advantages.view(-1)
    mean = (adv * mask).sum() / mask.sum()
    std = (((adv - mean) ** 2 * mask).sum() / mask.sum()).sqrt()
    adv = (adv - mean) / (std + 1e-8)
    old_logp, targets, actions = batch.logp.view(-1), batch.value_targets.view(-1), batch.actions.view(-1).long()
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(T * N, device=env.device)
        for k in range(0, T * N, args.minibatch):
            idx = perm[k:k + args.minibatch]
            rows = (2 * idx[:, None] + torch.arange(2, device=env.device)).view(-1)
            m = mask[rows]
            obs = batch.observations(idx).view(-1, W, H, 26).permute(0, 3, 1, 2)
            logits, value = model(obs)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(1, actions[rows, None]).squeeze(1)
            ratio = torch.exp(logp - old_logp[rows])
            a = adv[rows]
            masked_mean = lambda x: (x * m).sum() / m.sum().clamp(min=1)  # noqa: E731  the learner's rows only
            policy_loss = -masked_mean(torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a))
            value_loss = masked_mean((value - targets[rows]) ** 2)
            entropy = masked_mean(-(logp_all.exp() * logp_all).sum(-1))
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    sp.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  bc_factor %.3f  paired env-steps %.3f  shaping %.3f  episodes %d (with BC %d)  mean sparse return: with BC %.2f, "
          "self-play %.2f  policy loss %.4f  value loss %.3f  entropy %.3f  collect %.2f s  learn %.2f s"
          % (it, sp.bc_factor, paired, sp.reward_shaping_factor, episodes, int(with_bc.sum()), mean_return(with_bc),
             mean_return(~with_bc), policy_loss.item(), value_loss.item(), entropy.item(), t_collect, time.time() - t0), flush=True)
