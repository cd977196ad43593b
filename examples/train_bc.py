#!/usr/bin/env python
"""Behaviour cloning on the device: train K BC models (human_aware_rl's train_bc_model recipe) on recorded games and write
the first one's weights as the ``.npz`` that ``examples/ppo_bc.py --bc-weights`` reads.

The games are either played here, on the device, by two ``GreedyHumanModel`` agents (the reference's scripted partner),
or read from ``--games``: an ``.npz`` with ``states`` int32 [..., S] (the records each joint action was taken in) and
``actions`` int [..., 2] on ``--layout`` (e.g. tests/golden/greedy_cramped_room.npz, the reference's own greedy games;
reference trajectory dicts convert with ``wire.records_from_dicts`` and ``wire.action_indices``).  Each (transition,
player) is one training row: the player's featurize_state view and its action.  The trained policy then plays 400
transitions next to GreedyHumanModel.

    python examples/train_bc.py --out bc.npz
    python examples/train_bc.py --games tests/golden/greedy_cramped_room.npz --models 4 --out bc.npz
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200 import bc as B  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.greedy import GreedyHumanModel  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--layout", default="cramped_room")
ap.add_argument("--games", default=None, help=".npz of states / actions (default: greedy games played here)")
ap.add_argument("--envs", type=int, default=16, help="greedy games played at once")
ap.add_argument("--steps", type=int, default=400, help="transitions per greedy game")
ap.add_argument("--models", type=int, default=1)
ap.add_argument("--epochs", type=int, default=100)
ap.add_argument("--lr", type=float, default=1e-3)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--out", default="bc.npz")
args = ap.parse_args()

env = BatchedOvercookedEnv(args.layout, args.envs, horizon=400, auto_reset=True)
if args.games:
    z = np.load(args.games)
    records, actions = z["states"].reshape(-1, z["states"].shape[-1]), z["actions"].reshape(-1, 2)
else:
    pair = AgentPairRollout(env, (GreedyHumanModel(), GreedyHumanModel()), seed=args.seed, use_graph=False)
    recs, acts = [], []
    for _ in range(args.steps):
        recs.append(env.state.clone())
        pair.run(1)
        acts.append(pair.actions.view(-1, 2).clone())
    records, actions = torch.cat(recs), torch.cat(acts)
X, Y = B.bc_dataset(env, records, actions)
print("dataset: %d rows from %d transitions; action shares %s" % (X.shape[0], X.shape[0] // 2,
                                                                  np.round(np.bincount(Y.cpu().numpy(), minlength=6) / Y.numel(), 3)))
t0 = time.time()
models, history = B.train_bc(X, Y, n_models=args.models, seeds=[args.seed + k for k in range(args.models)], lr=args.lr,
                             epochs=args.epochs)
torch.cuda.synchronize()
print("trained %d models in %.2f s" % (args.models, time.time() - t0))
for k, h in enumerate(history):
    print("model %d: %d epochs, loss %.4f, accuracy %.4f, val loss %.4f, val accuracy %.4f, lr %.1e"
          % (k, len(h["loss"]), h["loss"][-1], h["accuracy"][-1], h["val_loss"][-1], h["val_accuracy"][-1], h["lr"][-1]))
B.save_keras_npz(models[0], args.out)
print("wrote", args.out)
play = BatchedOvercookedEnv(args.layout, 256, horizon=400, auto_reset=True)
evaluation = AgentPairRollout(play, (models[0], GreedyHumanModel()), seed=args.seed + 1)
evaluation.run(400)
ret = evaluation.episodes.finished()["ep_sparse_r"].float()
print("(BC, Greedy): mean sparse return %.2f over %d episodes" % (float(ret.mean()), ret.numel()))
