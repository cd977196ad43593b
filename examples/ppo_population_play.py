#!/usr/bin/env python
"""Population play (the PBT baseline of human-aware RL): K PPO agents that play each other, trained in ONE device rollout,
and the K x K cross-play matrix of a population.

``SelfPlayRollout(env, [m_0, ..., m_{K-1}], pair_weights=...)`` draws an ordered pair of members per episode (uniform
weights; ``--no-self-play`` zeroes the diagonal).  One ``collect()`` returns the ordinary two-view ``SampleBatch``; its
``pair`` says which member acted on each row, so member k trains, with its own Adam, on the flat rows where
``batch.pair.view(-1) == k``: row r is view ``r % 2`` of env-step ``r // 2``, evaluated by ``records_forward`` from the
stored record at that seat.  After each iteration ``sync_weights()`` refolds every member (the captured CUDA graph keeps
running) and the script prints the cross-play matrix of mean sparse returns of the episodes that ended, by their pair.
Checkpoints go to ``--save-dir/member_k.pt`` (``examples/ppo_population.py --members`` loads them).

``--evaluate DIR`` loads ``member_*.pt`` from DIR (this script's or ``ppo_selfplay_population.py``'s), gives each ordered
pair N / K^2 environments through fixed ``pairs``, runs whole episodes with ``run()`` and prints the matrix.  A
demonstration, not library code.

    python examples/ppo_population_play.py --k 4 --iters 5 --save-dir /tmp/pp
    python examples/ppo_population_play.py --evaluate /tmp/pp
"""
import argparse
import glob
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout, records_forward  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--k", type=int, default=4, help="population members")
ap.add_argument("--iters", type=int, default=5)
ap.add_argument("--envs", type=int, default=4096)
ap.add_argument("--steps", type=int, default=400)
ap.add_argument("--horizon", type=int, default=400)
ap.add_argument("--epochs", type=int, default=2)
ap.add_argument("--minibatch", type=int, default=8192, help="rows per minibatch of one member")
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--gamma", type=float, default=0.99)
ap.add_argument("--lam", type=float, default=0.98)
ap.add_argument("--clip", type=float, default=0.05)
ap.add_argument("--vf-coef", type=float, default=1e-4)
ap.add_argument("--entropy-coef", type=float, default=0.1)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--no-self-play", action="store_true", help="zero pair_weights' diagonal: members only meet other members")
ap.add_argument("--save-dir", default=None, help="write member_k.pt state dicts here")
ap.add_argument("--evaluate", default=None, help="a directory of member_*.pt: print their cross-play matrix and exit")
args = ap.parse_args()


def matrix(fin, K):
    """Mean sparse return per ordered pair (rows: the member on player 0) of the finished episodes ``fin``."""
    p, r = fin["pair"].cpu().numpy(), fin["ep_sparse_r"].float().cpu().numpy()
    m = np.full((K, K), np.nan)
    for i in range(K):
        for j in range(K):
            sel = (p[:, 0] == i) & (p[:, 1] == j)
            if sel.any():
                m[i, j] = r[sel].mean()
    return "\n".join("  p0=m%d  " % i + " ".join("%7.2f" % v for v in row) for i, row in enumerate(m))


if args.evaluate:
    paths = sorted(glob.glob(os.path.join(args.evaluate, "member_*.pt")), key=lambda s: int(s.rsplit("_", 1)[1][:-3]))
    K = len(paths)
    assert K >= 1, "no member_*.pt in %s" % args.evaluate
    q = max(args.envs // (K * K), 1)
    env = BatchedOvercookedEnv("cramped_room", K * K * q, horizon=args.horizon, auto_reset=True)
    W, H = env.layouts[0].width, env.layouts[0].height
    members = []
    for path in paths:
        m = RllibShapedCNN(W, H)
        m.load_state_dict(torch.load(path, map_location="cpu"))
        members.append(m.cuda())
    pairs = torch.tensor([(i, j) for i in range(K) for j in range(K)], dtype=torch.int32, device=env.device)
    sp = SelfPlayRollout(env, members, pairs=pairs.repeat_interleave(q, 0).contiguous(), seed=args.seed)
    sp.run(args.horizon)  # every environment ends exactly one episode
    print("cross-play of %d members (%d environments per ordered pair, mean sparse return):\n%s" % (K, q, matrix(sp.episodes.finished(), K)))
    sys.exit(0)

env = BatchedOvercookedEnv("cramped_room", args.envs, horizon=args.horizon, auto_reset=True)
W, H = env.layouts[0].width, env.layouts[0].height
members = []
for k in range(args.k):  # a different initialisation per member
    torch.manual_seed(args.seed * 1000 + k)
    members.append(RllibShapedCNN(W, H).cuda())
weights = np.ones((args.k, args.k))
if args.no_self_play:
    assert args.k > 1, "--no-self-play needs at least two members"
    np.fill_diagonal(weights, 0.0)
sp = SelfPlayRollout(env, members, pair_weights=weights, seed=args.seed)
opts = [torch.optim.Adam(m.parameters(), lr=args.lr) for m in members]
N, T, S = env.n_envs, args.steps, env.state_words
for it in range(args.iters):
    t0 = time.time()
    batch = sp.collect(T, args.gamma, args.lam)
    torch.cuda.synchronize()
    t_collect = time.time() - t0
    acting = batch.pair.view(-1).long()  # the member that acted on each flat row t * 2N + 2 e + v
    states = batch.states.view(-1, S)
    for k, (m, opt) in enumerate(zip(members, opts)):
        rows = torch.nonzero(acting == k).squeeze(1)
        if rows.numel() == 0:
            continue
        adv = batch.advantages.view(-1)[rows]
        adv = (adv - adv.mean()) / (adv.std() + 1e-8)
        old_logp, targets = batch.logp.view(-1)[rows], batch.value_targets.view(-1)[rows]
        actions = batch.actions.view(-1)[rows].long()
        for epoch in range(args.epochs):
            perm = torch.randperm(rows.numel(), device=env.device)
            for i in range(0, rows.numel(), args.minibatch):
                mb = perm[i:i + args.minibatch]
                r = rows[mb]
                swap = (r % 2).to(torch.int32).contiguous()  # seat 0 with swap = view: the row's own player
                logits, values = records_forward(m, env, states[r // 2].contiguous(), seat=0, swap=swap)
                logp_all = F.log_softmax(logits, -1)
                ratio = torch.exp(logp_all.gather(1, actions[mb, None]).squeeze(1) - old_logp[mb])
                pg = -torch.min(ratio * adv[mb], ratio.clamp(1 - args.clip, 1 + args.clip) * adv[mb]).mean()
                vf = F.mse_loss(values, targets[mb])
                ent = -(logp_all.exp() * logp_all).sum(-1).mean()
                loss = pg + args.vf_coef * vf - args.entropy_coef * ent
                opt.zero_grad()
                loss.backward()
                opt.step()
    sp.sync_weights()
    fin = batch.episodes.finished()
    print("iter %d  collect %.1f ms  %d episodes; cross-play (mean sparse return, row = member on player 0):\n%s"
          % (it, t_collect * 1e3, len(fin["env_index"]), matrix(fin, args.k)), flush=True)
if args.save_dir:
    os.makedirs(args.save_dir, exist_ok=True)
    for k, m in enumerate(members):
        torch.save(m.state_dict(), os.path.join(args.save_dir, "member_%d.pt" % k))
    print("saved %d members to %s (examples/ppo_population.py --members %s/member_*.pt)" % (args.k, args.save_dir, args.save_dir))
