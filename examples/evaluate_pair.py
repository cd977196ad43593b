#!/usr/bin/env python
"""The paper's evaluation on cramped_room (human_aware_rl's rllib.py ``evaluate``: AgentEvaluator.evaluate_agent_pair of
AgentPair(agent_0_policy, agent_1_policy)), with this library playing every game on the device:

  PPO against a behaviour-cloned "human proxy" in both seat orders (half of the environments swapped), one game per
  environment at horizon 400, the mean sparse return and its standard error per seat order;
  PPO_A against PPO_B (cross-play), the same statistics.

Each agent runs its own policy on its own seat's view only (AgentPairRollout).  Weights are random unless ``.npz`` files
of the reference's Keras arrays are given: ``--ppo-weights`` / ``--ppo-b-weights`` with ``conv_<i>_kernel`` / ``_bias``
(conv_initial, conv_0, conv_1), ``dense_<i>_kernel`` / ``_bias``, ``logits_*`` and ``value_*``; ``--bc-weights`` as
``examples/ppo_bc.py`` reads them.  A demonstration, not library code.

    python examples/evaluate_pair.py --envs 4096
"""
import argparse
import math
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from overcooked_ai_b200.batched import BatchedOvercookedEnv  # noqa: E402
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--envs", type=int, default=4096, help="games per pairing (one per environment)")
ap.add_argument("--horizon", type=int, default=400)
ap.add_argument("--ppo-weights", default=None)
ap.add_argument("--ppo-b-weights", default=None)
ap.add_argument("--bc-weights", default=None)
ap.add_argument("--seed", type=int, default=0)
args = ap.parse_args()
W, H = 5, 4


def ppo(path, seed):
    torch.manual_seed(seed)
    m = RllibShapedCNN(W, H)
    if path:
        z = np.load(path)
        n_dense = len([k for k in z.files if k.startswith("dense_") and k.endswith("_kernel")])
        m = RllibShapedCNN(W, H, num_hidden_layers=n_dense).load_keras_weights(
            [(z["conv_%d_kernel" % i], z["conv_%d_bias" % i]) for i in range(3)],
            [(z["dense_%d_kernel" % i], z["dense_%d_bias" % i]) for i in range(n_dense)],
            (z["logits_kernel"], z["logits_bias"]), (z["value_kernel"], z["value_bias"]))
    return m


def bc(path):
    if not path:
        return BCPolicy()
    z = np.load(path)
    n_dense = len([k for k in z.files if k.startswith("dense_") and k.endswith("_kernel")])
    return BCPolicy(num_hidden_layers=n_dense).load_keras_weights(
        [(z["dense_%d_kernel" % i], z["dense_%d_bias" % i]) for i in range(n_dense)], (z["logits_kernel"], z["logits_bias"]))


def play(agents, swap):
    """One game per environment; returns the sparse return of every game and the player agent 1 sat at."""
    env = BatchedOvercookedEnv(["cramped_room"], args.envs, horizon=args.horizon, auto_reset=True)
    pair = AgentPairRollout(env, agents, swap=swap, seed=args.seed)
    pair.run(args.horizon)
    fin = pair.episodes.finished()
    assert len(fin["ep_length"]) == args.envs
    return fin["ep_sparse_r"].cpu().numpy().astype(np.float64), fin["partner_seat"].cpu().numpy()


def report(name, r):
    print("%-34s games %6d  mean sparse return %7.2f  +- %.2f (standard error)" % (name, len(r), r.mean(), r.std(ddof=1) / math.sqrt(len(r))))


ppo_a, ppo_b, proxy = ppo(args.ppo_weights, 1), ppo(args.ppo_b_weights, 2), bc(args.bc_weights)
swap = (torch.arange(args.envs, device="cuda") % 2).to(torch.int32)  # half the games with the seats exchanged
ret, seat = play((ppo_a, proxy), swap)
report("PPO (player 0) x BC proxy", ret[seat == 1])
report("BC proxy (player 0) x PPO", ret[seat == 0])
ret, _ = play((ppo_a, ppo_b), None)
report("PPO_A x PPO_B (cross-play)", ret)
