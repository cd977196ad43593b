#!/usr/bin/env python
"""PPO self-play on cramped_room with this library as the rollout worker and a plain torch learner.

The worker (``SelfPlayRollout.collect``) runs the bf16 policy kernels K7 -> K9 -> K8 and the environments on the GPU
and returns a ``SampleBatch`` with behaviour log-probabilities, values, per-agent shaped rewards, dones and GAE
advantages.  The learner is torch autograd on ``RllibShapedCNN`` in float32 over observations re-encoded from the stored
records (``batch.observations``), with the clipped PPO objective and Adam.  ``--learner records`` trains the folded bf16
network the rollout runs instead, straight from the records (``batch.forward``: K7 forward, K12 weight gradient).  After each iteration ``sync_weights()``
folds the updated network back into the kernels' bf16 tables; the captured CUDA graph keeps running.

The behaviour policy is the bf16 fold of the learner's float32 weights, so the importance ratio is not exactly 1 even
at the first minibatch: the script prints max |ratio - 1| there to keep that mismatch visible.  A demonstration, not
library code: no entropy schedule, no KL penalty, one process.

    python examples/ppo_selfplay.py --iters 5
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.layout import EVENT_TYPES  # noqa: E402
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout  # noqa: E402

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
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--bootstrap-horizon", action="store_true",
                help="bootstrap the advantages from the value of each episode's last state at the horizon cut")
ap.add_argument("--use-phi", action="store_true", help="the potential-based dense reward (use_phi) instead of the shaped rewards")
ap.add_argument("--learner", choices=("conv", "records"), default="conv",
                help="conv: K2's float32 observation through RllibShapedCNN; records: batch.forward, the folded bf16 network "
                     "evaluated from the stored records (K7 forward, K12 for the first layer's weight gradient)")
args = ap.parse_args()

torch.manual_seed(args.seed)
env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=400, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
model = RllibShapedCNN(W, H).cuda()
sp = SelfPlayRollout(env, model=model, seed=args.seed, use_phi=args.use_phi)
opt = torch.optim.Adam(model.parameters(), lr=args.lr)
N, T = env.n_envs, args.steps
env_steps = 0
for it in range(args.iters):
    # the reference's linear annealing of the shaping factor (rllib.py:358-368), read by the captured graph
    sp.reward_shaping_factor = max(0.0, 1.0 - env_steps / args.shaping_horizon)
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam, bootstrap_horizon=args.bootstrap_horizon)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    # the episodes that ended in the window (TrainingCallbacks.on_episode_end's metrics, rllib.py:480-483)
    fin = batch.episodes.finished()
    episodes = fin["env_index"].numel()
    mean_sparse = float(fin["ep_sparse_r"].float().mean()) if episodes else float("nan")
    events = fin["ep_game_stats"].sum(1).float().mean(0) if episodes else torch.full((25,), float("nan"))
    event_means = "  ".join("%s %.2f" % (k, float(events[EVENT_TYPES.index(k)]))
                            for k in ("soup_delivery", "useful_onion_pickup", "optimal_onion_potting"))
    env_steps += T * N
    adv = batch.advantages.view(-1)
    adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    old_logp, targets, actions = batch.logp.view(-1), batch.value_targets.view(-1), batch.actions.view(-1).long()
    first_ratio = None
    t0 = time.time()
    for epoch in range(args.epochs):
        perm = torch.randperm(T * N, device=env.device)
        for k in range(0, T * N, args.minibatch):
            idx = perm[k:k + args.minibatch]
            rows = (2 * idx[:, None] + torch.arange(2, device=env.device)).view(-1)  # agent rows 2 (t N + e) + i
            if args.learner == "records":
                logits, value = batch.forward(model, idx)  # rows in the same order
            else:
                obs = batch.observations(idx).view(-1, W, H, 26).permute(0, 3, 1, 2)  # (2m, 26, W, H), agent order as rows
                logits, value = model(obs)
            logp_all = F.log_softmax(logits, dim=-1)
            logp = logp_all.gather(1, actions[rows, None]).squeeze(1)
            ratio = torch.exp(logp - old_logp[rows])
            if first_ratio is None:
                first_ratio = float((ratio.detach() - 1).abs().max())
            a = adv[rows]
            policy_loss = -torch.min(ratio * a, ratio.clamp(1 - args.clip, 1 + args.clip) * a).mean()
            value_loss = F.mse_loss(value, targets[rows])
            entropy = -(logp_all.exp() * logp_all).sum(-1).mean()
            loss = policy_loss + args.vf_coef * value_loss - args.entropy_coef * entropy
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
    sp.sync_weights()
    torch.cuda.synchronize()
    print("iter %d  shaping %.3f  episodes %d  mean sparse return %.2f  per episode: %s  first-minibatch max|ratio-1| %.4f  "
          "policy loss %.4f  value loss %.3f  entropy %.3f  collect %.2f s  learn %.2f s"
          % (it, sp.reward_shaping_factor, episodes, mean_sparse, event_means, first_ratio, policy_loss.item(), value_loss.item(),
             entropy.item(), t_collect, time.time() - t0), flush=True)
