"""Every rollout configuration against one host restatement of the rollout (tests/rollout_reference.py): the C oracle,
float64 networks and the documented draws.

``CONFIGURATIONS`` maps a case name to its value on each axis of ``AXES``; ``build`` turns those values into the
environment, the constructor arguments and the policy path the case claims.  tests/test_rollout_forms_cpu.py fails when a
value, or a pair of values of two axes, has no case (unless ``REFUSED`` names the test that shows the constructor refuses
it, or ``NOT_APPLICABLE`` says why it cannot occur), and when a constructor or collect() argument belongs to no axis.

Each case runs with and without CUDA graphs: two collect() windows (keep_logits in the second, both with the case's
bootstrap_horizon; between them the case's setters change and sync_weights() follows a second set of exact weights), every
batch field and the live state after each window against the reference, then run() one transition at a time (each joint
action checked) and the live state, the episode records and the counters again.  The kernels it launched must be the ones
its path names.  A staggered case starts a few environments part-way into their episodes, so that transitions end some
environments of a warp and not others.

Exactness: the network agents are ``P.exact_cnn`` models (distinct seeds per member; K7 -> library layers -> the draw kernel
runs on 5x5 grids), the BC agents ``_exact_bc``: every head and value is the float64 network's bit for bit, on the
bf16 and the float32 path alike (checked with certificates on the reference's layers before it is relied on).  LSTM agents
are seeded models with bf16-representable weights, compared within ``REPLAY_TOL`` and their draws checked where the Gumbel
gap exceeds the heads' bound."""
import re

import numpy as np
import pytest
import torch

import policy_reference as P
import rollout_reference as R
from oracle import cpu
from ppo_reference import gae_f32, gae_horizon_f32

GAMMA, LAM = 0.99, 0.95

# ---------------------------------------------------------------------------------------------------------- the axes
AXES = {
    "class": ["SelfPlayRollout", "AgentPairRollout"],
    "learner": ["cnn", "lstm", "blocks", "pairs", "pair_weights"],                       # SelfPlayRollout
    "partner": ["none", "bc", "cnn", "population_fixed", "population_drawn", "greedy"],  # SelfPlayRollout
    "bc_factor": ["0", "fraction", "1"],                                                 # SelfPlayRollout with a partner
    "agent0": ["cnn", "lstm", "bc", "greedy"],                                           # AgentPairRollout
    "agent1": ["cnn", "lstm", "bc", "population_fixed", "population_drawn", "greedy"],   # AgentPairRollout
    "seats": ["fixed", "swap", "random_seats"],                                          # AgentPairRollout
    "path": ["k7_k9_k8", "k7_library_draw", "k2_library_k8", "k2_library_draw", "float32", "learner_rows"],
    "starts": ["fixed", "random", "pool", "pool_redraw"],
    "use_phi": ["off", "on"],
    "episode_capacity": ["1", "2+"],
    "bootstrap_horizon": ["off", "on"],                                                  # collect()'s
    "phase": ["aligned", "staggered"],                                                   # the environments' timesteps
}
CLASS_AXES = {"SelfPlayRollout": ("learner", "partner", "bc_factor"), "AgentPairRollout": ("agent0", "agent1", "seats")}

# Every constructor argument of the two classes and the axis that covers it; every one of them is passed by some case
# (``passed_arguments``).
PARAMETERS = {
    "env": "starts", "model": "learner", "blocks": "learner", "pairs": "learner", "pair_weights": "learner",
    "partner": "partner", "member": "partner", "member_weights": "partner", "bc_factor": "bc_factor", "agents": "agent1",
    "swap": "seats", "random_seats": "seats", "autocast_dtype": "path", "fused_first_layer": "path", "fused_tail": "path",
    "fused_wide": "path", "use_phi": "use_phi", "episode_capacity": "episode_capacity",
}
# The arguments no axis varies, and why; every case passes them too.
NOT_AN_AXIS = {
    "use_graph": "every case runs with and without CUDA graphs",
    "seed": "every case draws from its own seed",
    "reward_shaping_factor": "every case sets it, and changes it between its windows",
    "max_seq_len": "every LSTM case cuts its windows into chunks that episodes end inside and at",
}
# Every argument of collect() and the axis that covers it, or why no axis varies it.
COLLECT_PARAMETERS = {"bootstrap_horizon": "bootstrap_horizon"}
COLLECT_NOT_AN_AXIS = {
    "n_steps": "every case collects windows of its own length T, longer than its horizon",
    "gamma": "every case uses the same gamma: GAE's arithmetic is checked bit for bit, not its constants",
    "lam": "every case uses the same lambda: GAE's arithmetic is checked bit for bit, not its constants",
    "keep_logits": "every case collects its first window without and its second with keep_logits",
}

PARTNERS = ("bc", "cnn", "population_fixed", "population_drawn", "greedy")
HORIZON_REFUSED = "test_horizon_bootstrap_cpu.py::test_refused_configurations"
SCRIPTED = ("bc", "greedy")  # agents without a network

# (axis, value, axis, value, the existing CPU test that asserts the constructor refuses the pair)
REFUSED = [
    ("learner", "lstm", "path", "float32", "test_rollout_forms_cpu.py::test_selfplay_refuses_a_float32_lstm_learner"),
    ("agent0", "lstm", "path", "float32", "test_agent_pair_cpu.py::test_agent_pair_refuses_mixed_grids_and_a_float32_lstm_agent"),
    ("agent1", "lstm", "path", "float32", "test_rollout_forms_cpu.py::test_agent_pair_refuses_a_float32_lstm_agent_1"),
    ("learner", "blocks", "partner", PARTNERS, "test_selfplay_population_cpu.py::test_selfplay_refuses_a_malformed_population_of_learners"),
    ("learner", "pairs", "partner", PARTNERS, "test_population_play_cpu.py::test_selfplay_refuses_population_play_with_what_it_excludes"),
    ("learner", "pair_weights", "partner", PARTNERS, "test_population_play_cpu.py::test_selfplay_refuses_population_play_with_what_it_excludes"),
    ("learner", "pairs", "path", "float32", "test_population_play_cpu.py::test_selfplay_refuses_population_play_with_what_it_excludes"),
    ("learner", "pair_weights", "path", "float32", "test_population_play_cpu.py::test_selfplay_refuses_population_play_with_what_it_excludes"),
    ("learner", "pairs", "path", "k2_library_k8", "test_population_play_cpu.py::test_selfplay_refuses_population_play_beyond_k7"),
    ("learner", "pair_weights", "path", "k2_library_k8", "test_population_play_cpu.py::test_selfplay_refuses_population_play_beyond_k7"),
    ("learner", "pairs", "path", "k2_library_draw", "test_rollout_forms_cpu.py::test_selfplay_refuses_population_play_on_a_9x5_grid"),
    ("learner", "pair_weights", "path", "k2_library_draw", "test_rollout_forms_cpu.py::test_selfplay_refuses_population_play_on_a_9x5_grid"),
    ("bootstrap_horizon", "on", "learner", ("lstm", "blocks", "pairs", "pair_weights"), HORIZON_REFUSED),
    ("bootstrap_horizon", "on", "agent0", "lstm", HORIZON_REFUSED),
]

# (axis, value, axis, value, why the pair cannot occur); a value may be "*" (every value) or a tuple of values
NOT_APPLICABLE = [
    ("class", "SelfPlayRollout", "agent0", "*", "agents are AgentPairRollout's"),
    ("class", "SelfPlayRollout", "agent1", "*", "agents are AgentPairRollout's"),
    ("class", "SelfPlayRollout", "seats", "*", "a SelfPlayRollout's seats are its partner's seat draw (the bc_factor axis)"),
    ("class", "AgentPairRollout", "learner", "*", "an AgentPairRollout's learner is agent 0"),
    ("class", "AgentPairRollout", "partner", "*", "an AgentPairRollout's partner is agent 1"),
    ("class", "AgentPairRollout", "bc_factor", "*", "an AgentPairRollout's agent 1 plays every episode"),
    ("class", "AgentPairRollout", "path", "learner_rows", "learner rows are a self-play mixture's"),
    ("partner", "none", "bc_factor", "*", "bc_factor weighs the partner's episodes"),
    ("partner", "none", "path", "learner_rows", "the learner runs on its own rows only next to a network partner"),
    ("partner", "bc", "path", "learner_rows", "the learner runs on its own rows only next to a network partner"),
    ("partner", "greedy", "path", "learner_rows", "the learner runs on its own rows only next to a network partner"),
    ("learner", "lstm", "path", "learner_rows", "an LSTM learner runs on all 2N rows (K11 has no rows form)"),
    ("learner", "blocks", "path", "learner_rows", "the learner runs on its own rows only next to a partner"),
    ("learner", "pairs", "path", "learner_rows", "the learner runs on its own rows only next to a partner"),
    ("learner", "pair_weights", "path", "learner_rows", "the learner runs on its own rows only next to a partner"),
    ("path", "k2_library_k8", "starts", "fixed", "K2 -> library -> K8 runs on 5x4 pools of more than 8 layouts only"),
    ("path", "k2_library_k8", "starts", "random", "K2 -> library -> K8 runs on 5x4 pools of more than 8 layouts only"),
    ("agent0", SCRIPTED, "agent1", SCRIPTED, "a BC or greedy agent against another evaluates no network: no path to claim"),
    ("bootstrap_horizon", "on", "agent0", SCRIPTED, "a BC or greedy agent 0 has no collect(), so no bootstrap"),
    ("agent0", "*", "path", "learner_rows", "learner rows are a self-play mixture's"),
    ("agent1", "*", "path", "learner_rows", "learner rows are a self-play mixture's"),
    ("seats", "*", "path", "learner_rows", "learner rows are a self-play mixture's"),
    ("learner", ("blocks", "pairs", "pair_weights"), "bc_factor", "*", "a population of learners has no partner"),
] + [(a, "*", b, "*", "one axis is SelfPlayRollout's, the other AgentPairRollout's")
     for a in CLASS_AXES["SelfPlayRollout"] for b in CLASS_AXES["AgentPairRollout"]]

# the cases: each value of every axis of its class and of the shared axes; sizes N, T, horizon and the LSTM's chunk.  The
# sizes are free, with one constraint: pair_cnn_lstm_random_seats_k7_k9_k8_pool_phi1_cap2_bh1 runs at horizon 12, because
# at 13 environment 0's LSTM agent 1 meets a near-tie at its episode's last step between picking up a dish and an action
# that leaves the same reset record and reward; the reference cannot tell them apart (_settle), and the dish pickup shows
# only in the episode's game statistics.
CONFIGURATIONS = {
    "sp_lstm_cnn_bcf_k2_library_draw_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "cnn", "bc_factor": "fraction", "path": "k2_library_draw", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 97, "T": 17, "horizon": 7},
    "pair_lstm_cnn_random_seats_k7_library_draw_pool_phi1_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "cnn", "seats": "random_seats", "path": "k7_library_draw", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 101, "T": 18, "horizon": 8},
    "sp_cnn_population_drawn_bc0_float32_fixed_phi1_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_drawn", "bc_factor": "0", "path": "float32", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 103, "T": 19, "horizon": 9},
    "pair_cnn_lstm_swap_k7_k9_k8_fixed_phi0_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "lstm", "seats": "swap", "path": "k7_k9_k8", "starts": "fixed", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 107, "T": 17, "horizon": 10},
    "pair_bc_population_fixed_fixed_k2_library_k8_pool_redraw_phi1_cap2": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "population_fixed", "seats": "fixed", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 109, "T": 18, "horizon": 11},
    "sp_cnn_population_fixed_bc1_learner_rows_random_phi0_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_fixed", "bc_factor": "1", "path": "learner_rows", "starts": "random", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 113, "T": 19, "horizon": 12},
    "pair_bc_population_drawn_random_seats_float32_random_phi0_cap1": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "population_drawn", "seats": "random_seats", "path": "float32", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 115, "T": 17, "horizon": 13},
    "sp_lstm_bc_bc1_k2_library_k8_pool_phi1_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "bc", "bc_factor": "1", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 117, "T": 18, "horizon": 7},
    "pair_cnn_bc_swap_k2_library_draw_random_phi1_cap2": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "bc", "seats": "swap", "path": "k2_library_draw", "starts": "random", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 119, "T": 19, "horizon": 8},
    "pair_lstm_bc_fixed_k7_library_draw_fixed_phi0_cap1": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "bc", "seats": "fixed", "path": "k7_library_draw", "starts": "fixed", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 121, "T": 17, "horizon": 9},
    "sp_lstm_population_fixed_bcf_k7_k9_k8_pool_phi1_cap2": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "population_fixed", "bc_factor": "fraction", "path": "k7_k9_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 123, "T": 18, "horizon": 10},
    "sp_lstm_population_drawn_bc0_k7_library_draw_random_phi0_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "population_drawn", "bc_factor": "0", "path": "k7_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 125, "T": 19, "horizon": 11},
    "sp_blocks_none_k2_library_draw_pool_phi0_cap1": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "k2_library_draw", "starts": "pool", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 127, "T": 17, "horizon": 12},
    "sp_cnn_cnn_bc0_learner_rows_pool_phi1_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "0", "path": "learner_rows", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 97, "T": 18, "horizon": 13},
    "sp_pairs_none_k7_k9_k8_random_phi1_cap2": {"class": "SelfPlayRollout", "learner": "pairs", "partner": "none", "path": "k7_k9_k8", "starts": "random", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 101, "T": 19, "horizon": 7},
    "pair_cnn_cnn_random_seats_k2_library_k8_pool_redraw_phi0_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "cnn", "seats": "random_seats", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 103, "T": 17, "horizon": 8},
    "pair_lstm_population_drawn_swap_k7_library_draw_pool_redraw_phi1_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "population_drawn", "seats": "swap", "path": "k7_library_draw", "starts": "pool_redraw", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 107, "T": 18, "horizon": 9},
    "sp_cnn_bc_bc0_k7_k9_k8_pool_redraw_phi0_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "bc", "bc_factor": "0", "path": "k7_k9_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 109, "T": 19, "horizon": 10},
    "pair_cnn_population_fixed_swap_float32_pool_phi0_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "population_fixed", "seats": "swap", "path": "float32", "starts": "pool", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 113, "T": 17, "horizon": 11},
    "pair_lstm_lstm_fixed_k2_library_draw_random_phi1_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "lstm", "seats": "fixed", "path": "k2_library_draw", "starts": "random", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 115, "T": 18, "horizon": 12},
    "sp_pair_weights_none_k7_library_draw_fixed_phi1_cap2": {"class": "SelfPlayRollout", "learner": "pair_weights", "partner": "none", "path": "k7_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 117, "T": 19, "horizon": 13},
    "pair_bc_cnn_swap_k2_library_draw_fixed_phi1_cap1": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "cnn", "seats": "swap", "path": "k2_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 119, "T": 17, "horizon": 7},
    "pair_bc_population_drawn_fixed_k7_k9_k8_pool_phi0_cap2": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "population_drawn", "seats": "fixed", "path": "k7_k9_k8", "starts": "pool", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 121, "T": 18, "horizon": 8},
    "sp_cnn_cnn_bcf_k7_library_draw_random_phi0_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "fraction", "path": "k7_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 123, "T": 19, "horizon": 9},
    "sp_blocks_none_float32_pool_redraw_phi1_cap2": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "float32", "starts": "pool_redraw", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 125, "T": 17, "horizon": 10},
    "pair_lstm_population_fixed_random_seats_k7_k9_k8_fixed_phi0_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "population_fixed", "seats": "random_seats", "path": "k7_k9_k8", "starts": "fixed", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 127, "T": 18, "horizon": 11},
    "sp_cnn_population_fixed_bc0_k2_library_draw_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_fixed", "bc_factor": "0", "path": "k2_library_draw", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 97, "T": 19, "horizon": 12},
    "sp_lstm_cnn_bc1_k7_k9_k8_fixed_phi0_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "cnn", "bc_factor": "1", "path": "k7_k9_k8", "starts": "fixed", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 101, "T": 17, "horizon": 13},
    "pair_bc_lstm_random_seats_k7_library_draw_pool_phi0_cap2": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "lstm", "seats": "random_seats", "path": "k7_library_draw", "starts": "pool", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 103, "T": 18, "horizon": 7},
    "sp_cnn_population_drawn_bcf_k2_library_k8_pool_phi1_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_drawn", "bc_factor": "fraction", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 107, "T": 19, "horizon": 8},
    "pair_cnn_cnn_fixed_float32_random_phi0_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "cnn", "seats": "fixed", "path": "float32", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 109, "T": 17, "horizon": 9},
    "sp_cnn_bc_bcf_float32_fixed_phi0_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "bc", "bc_factor": "fraction", "path": "float32", "starts": "fixed", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 113, "T": 18, "horizon": 10},
    "sp_lstm_population_drawn_bc1_k2_library_draw_pool_redraw_phi1_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "population_drawn", "bc_factor": "1", "path": "k2_library_draw", "starts": "pool_redraw", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 115, "T": 19, "horizon": 11},
    "pair_lstm_bc_swap_k2_library_k8_pool_redraw_phi0_cap1": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "bc", "seats": "swap", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 117, "T": 17, "horizon": 12},
    "sp_pair_weights_none_k7_k9_k8_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "pair_weights", "partner": "none", "path": "k7_k9_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 119, "T": 18, "horizon": 13},
    "sp_pairs_none_k7_library_draw_pool_phi0_cap1": {"class": "SelfPlayRollout", "learner": "pairs", "partner": "none", "path": "k7_library_draw", "starts": "pool", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 121, "T": 19, "horizon": 7},
    "pair_cnn_population_drawn_random_seats_k2_library_draw_fixed_phi1_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "population_drawn", "seats": "random_seats", "path": "k2_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 123, "T": 17, "horizon": 8},
    "sp_lstm_bc_bc1_k7_library_draw_random_phi0_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "bc", "bc_factor": "1", "path": "k7_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 125, "T": 18, "horizon": 9},
    "sp_cnn_population_fixed_bc1_float32_fixed_phi1_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_fixed", "bc_factor": "1", "path": "float32", "starts": "fixed", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 127, "T": 19, "horizon": 10},
    "sp_cnn_population_drawn_bcf_learner_rows_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_drawn", "bc_factor": "fraction", "path": "learner_rows", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 97, "T": 17, "horizon": 11},
    "pair_cnn_population_fixed_swap_k7_library_draw_random_phi0_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "population_fixed", "seats": "swap", "path": "k7_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 101, "T": 18, "horizon": 12},
    "pair_cnn_bc_random_seats_float32_pool_phi1_cap1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "bc", "seats": "random_seats", "path": "float32", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 103, "T": 19, "horizon": 13},
    "sp_blocks_none_k7_library_draw_fixed_phi1_cap2": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "k7_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 107, "T": 17, "horizon": 7},
    "sp_cnn_population_fixed_bc0_k2_library_k8_pool_phi0_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_fixed", "bc_factor": "0", "path": "k2_library_k8", "starts": "pool", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 109, "T": 18, "horizon": 8},
    "pair_lstm_lstm_fixed_k2_library_k8_pool_redraw_phi0_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "lstm", "seats": "fixed", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 113, "T": 19, "horizon": 9},
    "sp_blocks_none_k2_library_k8_pool_phi1_cap1": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 115, "T": 17, "horizon": 10},
    "sp_blocks_none_k7_k9_k8_random_phi1_cap2": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "k7_k9_k8", "starts": "random", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 117, "T": 18, "horizon": 11},
    "sp_lstm_bc_bcf_k2_library_draw_pool_phi1_cap2": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "bc", "bc_factor": "fraction", "path": "k2_library_draw", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 119, "T": 19, "horizon": 12},
    "sp_cnn_cnn_bc1_float32_pool_phi1_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "1", "path": "float32", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 121, "T": 17, "horizon": 13},
    "sp_pairs_none_k7_k9_k8_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "pairs", "partner": "none", "path": "k7_k9_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 123, "T": 18, "horizon": 7},
    "pair_lstm_population_drawn_fixed_k2_library_k8_pool_phi1_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "population_drawn", "seats": "fixed", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 125, "T": 19, "horizon": 8},
    "sp_lstm_population_fixed_bc0_k7_library_draw_pool_phi0_cap2": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "population_fixed", "bc_factor": "0", "path": "k7_library_draw", "starts": "pool", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 127, "T": 17, "horizon": 9},
    "pair_bc_cnn_random_seats_k7_k9_k8_pool_phi1_cap1": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "cnn", "seats": "random_seats", "path": "k7_k9_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 97, "T": 18, "horizon": 10},
    "pair_bc_population_fixed_random_seats_k2_library_draw_random_phi0_cap2": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "population_fixed", "seats": "random_seats", "path": "k2_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 101, "T": 19, "horizon": 11},
    "sp_lstm_none_k2_library_k8_pool_phi1_cap2": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "none", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 103, "T": 17, "horizon": 12},
    "pair_lstm_bc_random_seats_k7_k9_k8_fixed_phi0_cap2": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "bc", "seats": "random_seats", "path": "k7_k9_k8", "starts": "fixed", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 107, "T": 18, "horizon": 13},
    "sp_cnn_cnn_bc1_k2_library_k8_pool_redraw_phi0_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "1", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 109, "T": 19, "horizon": 7},
    "sp_cnn_none_k2_library_draw_fixed_phi1_cap2": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "none", "path": "k2_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "aligned", "n": 113, "T": 17, "horizon": 8},
    "sp_cnn_cnn_bc1_learner_rows_fixed_phi1_cap1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "1", "path": "learner_rows", "starts": "fixed", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 115, "T": 18, "horizon": 9},
    "sp_lstm_population_drawn_bcf_k7_k9_k8_fixed_phi0_cap1": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "population_drawn", "bc_factor": "fraction", "path": "k7_k9_k8", "starts": "fixed", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 117, "T": 19, "horizon": 10},
    "sp_pairs_none_k7_library_draw_fixed_phi1_cap1": {"class": "SelfPlayRollout", "learner": "pairs", "partner": "none", "path": "k7_library_draw", "starts": "fixed", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 119, "T": 17, "horizon": 11},
    "sp_pair_weights_none_k7_library_draw_pool_phi1_cap1": {"class": "SelfPlayRollout", "learner": "pair_weights", "partner": "none", "path": "k7_library_draw", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 121, "T": 18, "horizon": 12},
    "sp_pair_weights_none_k7_library_draw_random_phi1_cap1": {"class": "SelfPlayRollout", "learner": "pair_weights", "partner": "none", "path": "k7_library_draw", "starts": "random", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 123, "T": 19, "horizon": 13},
    "sp_cnn_greedy_bcf_k7_library_draw_pool_redraw_phi0_cap2_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "greedy", "bc_factor": "fraction", "path": "k7_library_draw", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "staggered", "n": 125, "T": 17, "horizon": 7},
    "pair_cnn_greedy_fixed_k7_k9_k8_pool_phi1_cap1_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "greedy", "seats": "fixed", "path": "k7_k9_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 127, "T": 18, "horizon": 8},
    "pair_greedy_cnn_swap_float32_fixed_phi1_cap2_stag": {"class": "AgentPairRollout", "agent0": "greedy", "agent1": "cnn", "seats": "swap", "path": "float32", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "staggered", "n": 97, "T": 19, "horizon": 9},
    "pair_greedy_population_drawn_random_seats_k7_k9_k8_random_phi0_cap1_stag": {"class": "AgentPairRollout", "agent0": "greedy", "agent1": "population_drawn", "seats": "random_seats", "path": "k7_k9_k8", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 101, "T": 17, "horizon": 10},
    "pair_cnn_greedy_random_seats_k7_library_draw_pool_redraw_phi0_cap2_bh1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "greedy", "seats": "random_seats", "path": "k7_library_draw", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "aligned", "n": 103, "T": 18, "horizon": 11},
    "sp_lstm_greedy_bc1_k2_library_k8_pool_phi1_cap1_stag": {"class": "SelfPlayRollout", "learner": "lstm", "partner": "greedy", "bc_factor": "1", "path": "k2_library_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 107, "T": 19, "horizon": 12},
    "sp_cnn_greedy_bc0_k2_library_draw_random_phi1_cap1_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "greedy", "bc_factor": "0", "path": "k2_library_draw", "starts": "random", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 109, "T": 17, "horizon": 13},
    "pair_greedy_lstm_fixed_k2_library_k8_pool_redraw_phi0_cap2_stag": {"class": "AgentPairRollout", "agent0": "greedy", "agent1": "lstm", "seats": "fixed", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "staggered", "n": 113, "T": 18, "horizon": 7},
    "pair_greedy_population_fixed_swap_k2_library_draw_random_phi0_cap1_stag": {"class": "AgentPairRollout", "agent0": "greedy", "agent1": "population_fixed", "seats": "swap", "path": "k2_library_draw", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 115, "T": 19, "horizon": 8},
    "sp_cnn_greedy_bc1_float32_fixed_phi1_cap2_bh1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "greedy", "bc_factor": "1", "path": "float32", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "aligned", "n": 117, "T": 17, "horizon": 9},
    "sp_cnn_greedy_bcf_k7_k9_k8_pool_redraw_phi0_cap1_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "greedy", "bc_factor": "fraction", "path": "k7_k9_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 119, "T": 18, "horizon": 10},
    "pair_cnn_greedy_swap_float32_random_phi0_cap1_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "greedy", "seats": "swap", "path": "float32", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 121, "T": 19, "horizon": 11},
    "pair_lstm_greedy_random_seats_k2_library_k8_pool_redraw_phi0_cap1_stag": {"class": "AgentPairRollout", "agent0": "lstm", "agent1": "greedy", "seats": "random_seats", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 123, "T": 17, "horizon": 12},
    "pair_greedy_population_drawn_random_seats_k7_library_draw_pool_phi1_cap1": {"class": "AgentPairRollout", "agent0": "greedy", "agent1": "population_drawn", "seats": "random_seats", "path": "k7_library_draw", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "aligned", "n": 125, "T": 18, "horizon": 13},
    "pair_cnn_greedy_fixed_k2_library_draw_fixed_phi0_cap2_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "greedy", "seats": "fixed", "path": "k2_library_draw", "starts": "fixed", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "staggered", "n": 127, "T": 19, "horizon": 7},
    "sp_cnn_cnn_bc1_learner_rows_pool_phi0_cap2_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "cnn", "bc_factor": "1", "path": "learner_rows", "starts": "pool", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "staggered", "n": 97, "T": 17, "horizon": 8},
    "sp_cnn_population_fixed_bcf_k2_library_k8_pool_redraw_phi0_cap1_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_fixed", "bc_factor": "fraction", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 101, "T": 18, "horizon": 9},
    "sp_pairs_none_k7_k9_k8_random_phi1_cap2_stag": {"class": "SelfPlayRollout", "learner": "pairs", "partner": "none", "path": "k7_k9_k8", "starts": "random", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "staggered", "n": 103, "T": 19, "horizon": 10},
    "sp_cnn_bc_bcf_k7_k9_k8_pool_redraw_phi1_cap1_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "bc", "bc_factor": "fraction", "path": "k7_k9_k8", "starts": "pool_redraw", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 107, "T": 17, "horizon": 11},
    "pair_cnn_bc_random_seats_float32_pool_phi1_cap2_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "bc", "seats": "random_seats", "path": "float32", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "staggered", "n": 109, "T": 18, "horizon": 12},
    "sp_cnn_population_drawn_bcf_k7_library_draw_pool_redraw_phi0_cap1_bh1_stag": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "population_drawn", "bc_factor": "fraction", "path": "k7_library_draw", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 113, "T": 19, "horizon": 13},
    "sp_blocks_none_k2_library_k8_pool_redraw_phi0_cap1_stag": {"class": "SelfPlayRollout", "learner": "blocks", "partner": "none", "path": "k2_library_k8", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 115, "T": 17, "horizon": 7},
    "pair_bc_cnn_swap_float32_pool_phi1_cap2_stag": {"class": "AgentPairRollout", "agent0": "bc", "agent1": "cnn", "seats": "swap", "path": "float32", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "off", "phase": "staggered", "n": 117, "T": 18, "horizon": 8},
    "pair_cnn_cnn_fixed_k7_k9_k8_random_phi0_cap1_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "cnn", "seats": "fixed", "path": "k7_k9_k8", "starts": "random", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "staggered", "n": 119, "T": 19, "horizon": 9},
    "sp_cnn_none_float32_fixed_phi1_cap2_bh1": {"class": "SelfPlayRollout", "learner": "cnn", "partner": "none", "path": "float32", "starts": "fixed", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "aligned", "n": 121, "T": 17, "horizon": 10},
    "pair_cnn_population_fixed_random_seats_float32_fixed_phi0_cap2_bh1_stag": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "population_fixed", "seats": "random_seats", "path": "float32", "starts": "fixed", "use_phi": "off", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "staggered", "n": 123, "T": 18, "horizon": 11},
    "pair_cnn_population_drawn_swap_float32_pool_redraw_phi0_cap1_bh1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "population_drawn", "seats": "swap", "path": "float32", "starts": "pool_redraw", "use_phi": "off", "episode_capacity": "1", "bootstrap_horizon": "on", "phase": "aligned", "n": 125, "T": 19, "horizon": 12},
    "pair_cnn_lstm_random_seats_k7_k9_k8_pool_phi1_cap2_bh1": {"class": "AgentPairRollout", "agent0": "cnn", "agent1": "lstm", "seats": "random_seats", "path": "k7_k9_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "2+", "bootstrap_horizon": "on", "phase": "aligned", "n": 127, "T": 17, "horizon": 12},
    "sp_pair_weights_none_k7_k9_k8_pool_phi1_cap1_stag": {"class": "SelfPlayRollout", "learner": "pair_weights", "partner": "none", "path": "k7_k9_k8", "starts": "pool", "use_phi": "on", "episode_capacity": "1", "bootstrap_horizon": "off", "phase": "staggered", "n": 97, "T": 18, "horizon": 7},
}


# ---------------------------------------------------------------------------------------------------------- building
def _pool_5x4():
    from test_gpu_bc_partner import POOL_5X4
    return POOL_5X4


GRIDS = {  # path -> (the single layout, the pool); K2 -> library -> K8 needs more than 8 5x4 layouts, so K7 is off
    "k7_k9_k8": ("cramped_room", ["cramped_room", "mdp_test", "bonus_order_test", "simple_o"]),
    "learner_rows": ("cramped_room", ["cramped_room", "mdp_test", "bonus_order_test", "simple_o"]),
    "float32": ("cramped_room", ["cramped_room", "mdp_test", "bonus_order_test", "simple_o"]),
    "k7_library_draw": ("coordination_ring", ["coordination_ring", "forced_coordination", "five_by_five"]),
    "k2_library_k8": (None, None),
    "k2_library_draw": ("asymmetric_advantages", ["asymmetric_advantages", "counter_circuit", "cramped_corridor"]),
}
# A case with a greedy agent plays layouts of one 3-onion order only (GreedyHumanModel's ml_action asserts it): mdp_test,
# bonus_order_test, counter_circuit and cramped_corridor do not qualify.  Nine 5x4 layouts (duplicates allowed) turn K7 off
# for K2 -> library -> K8; on the 9x5 grid only asymmetric_advantages qualifies, so no pool there.
GREEDY_POOL_5X4 = ["cramped_room", "m_shaped_s", "simple_o"]
GREEDY_GRIDS = {
    "k7_k9_k8": ("cramped_room", GREEDY_POOL_5X4),
    "float32": ("cramped_room", GREEDY_POOL_5X4),
    "k7_library_draw": GRIDS["k7_library_draw"],
    "k2_library_k8": (None, GREEDY_POOL_5X4 * 3),
    "k2_library_draw": ("asymmetric_advantages", None),
}
BC_FACTOR = {"0": 0.0, "fraction": 0.6, "1": 1.0}
BC_FACTOR_LATER = {"0": 0.5, "fraction": 0.25, "1": 0.8}
WEIGHTS, WEIGHTS_LATER = [1.0, 2.0, 0.5], [0.5, 0.0, 2.0]
PAIR_WEIGHTS = [[0.0, 1.0, 2.0], [1.0, 0.5, 1.0], [3.0, 1.0, 0.0]]
PAIR_WEIGHTS_LATER = [[1.0, 0.0, 0.0], [0.0, 0.0, 2.0], [1.0, 1.0, 1.0]]
SEQ_LEN = 4
# SelfPlayRollout's (fused_first_layer, fused_tail, fused_wide) for each path, passed explicitly so that a case's path is
# its arguments, not only their defaults (AgentPairRollout takes no such arguments: its agents follow the defaults)
FUSED = {"k7_k9_k8": (True, True, True), "learner_rows": (True, True, True), "k7_library_draw": (True, False, False),
         "k2_library_k8": (False, True, False), "k2_library_draw": (False, False, False), "float32": (False, False, False)}


def is_greedy(case):
    return "greedy" in (case.get("partner"), case.get("agent0"), case.get("agent1"))


def staggered_timesteps(n, horizon):
    """The staggered phase's starting timesteps: 0 but for one environment in each warp of 32 from the second on, at
    horizon - 1 in odd warps (its episode ends alone at the first transition, where the start it resets to is the one it
    played from) and at horizon // 2 in even ones.  The first warp, and every warp at its common horizon, ends every
    environment at once; the others end one environment alone, or all but one."""
    t = np.zeros(n, np.int32)
    for w in range(1, -(-n // 32)):
        t[32 * w + (7 * w) % min(32, n - 32 * w)] = horizon - 1 if w % 2 else horizon // 2
    return t


def passed_arguments(case):
    """The constructor arguments ``build`` passes for a case (by keyword, ``env`` and ``model`` / ``agents`` too)."""
    out = {"env", "use_graph", "seed", "episode_capacity", "use_phi", "max_seq_len"}
    if case["path"] == "float32":
        out.add("autocast_dtype")
    if case["class"] == "SelfPlayRollout":
        out |= {"model", "reward_shaping_factor", "fused_first_layer", "fused_tail", "fused_wide"}
        out |= {"blocks": {"blocks"}, "pairs": {"pairs"}, "pair_weights": {"pair_weights"}}.get(case["learner"], set())
        owner = case["partner"]
        if owner != "none":
            out |= {"partner", "bc_factor"}
    else:
        out.add("agents")
        owner = case["agent1"]
        out |= {"swap": {"swap"}, "random_seats": {"random_seats"}}.get(case["seats"], set())
    out |= {"population_fixed": {"member"}, "population_drawn": {"member_weights"}}.get(owner, set())
    return out


def _env(case, seed):
    """(env, cpu.random_start or None) of the case's starts on the grid its path runs on, at the case's phase."""
    from overcooked_ai_b200.batched import BatchedOvercookedEnv

    single, pool = (GREEDY_GRIDS if is_greedy(case) else GRIDS)[case["path"]]
    if pool is None and not is_greedy(case):
        pool = _pool_5x4()
    n, st = case["n"], case["starts"]
    kw = dict(horizon=case["horizon"], auto_reset=True)
    rs = None
    if st == "fixed":
        layouts = single
    elif st == "random":
        layouts = single
        kw.update(random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=seed)
        rs = cpu.random_start(seed, 0.5, True, False)
    elif st == "pool":
        layouts = pool
        kw.update(env_layout=np.arange(n) % len(pool))
    else:
        layouts = pool
        kw.update(random_layout=True, seed=seed)
        rs = cpu.random_start(seed, 0.0, False, True)
    env = BatchedOvercookedEnv(layouts, n, **kw)
    if case["phase"] == "staggered":  # word 0 of a record is its timestep (DESIGN §3)
        env.state[:, 0] = torch.from_numpy(staggered_timesteps(n, case["horizon"])).to(env.device)
    return env, rs


def _host(env, rs, use_phi):
    from overcooked_ai_b200 import layout as L

    lut = np.stack([l.feature_lut() for l in env.layouts]).view(np.uint8).reshape(env.n_layouts, -1)
    pot = L.build_potential_tables(env.layouts, R.PHI_GAMMA) if use_phi else None
    return R.EnvHost(env._tab_host, env._starts_host, env.horizon, rs, env.layouts[0].width, env.layouts[0].height, lut, pot,
                     np.stack([l.deliver_value for l in env.layouts]), env.n_envs, env.layouts)


class _Models(object):
    """The case's models by role, each exact (or, for the LSTM, bf16-representable); ``second()`` loads a second set of
    weights into the same objects."""

    def __init__(self, env):
        self.W, self.H, self.cook = env.layouts[0].width, env.layouts[0].height, env._longest_cook
        self.made = []

    def _weights(self, kind, seed, head_scale=30.0):
        from test_gpu_bc_partner import _exact_bc
        from overcooked_ai_b200.greedy import GreedyHumanModel
        from overcooked_ai_b200.selfplay import RllibLSTMShapedCNN

        if kind == "greedy":
            return GreedyHumanModel()
        if kind == "cnn":
            return P.exact_cnn(self.W, self.H, seed, cook_time=self.cook)
        if kind == "bc":
            return _exact_bc(np.random.RandomState(seed))[0]
        torch.manual_seed(seed)
        m = RllibLSTMShapedCNN(self.W, self.H)
        with torch.no_grad():
            m.logits.weight.mul_(head_scale), m.value.weight.mul_(head_scale)
            for p_ in m.parameters():
                p_.copy_(p_.bfloat16().float())
        return m

    def make(self, kind, seed, head_scale=30.0):
        """``head_scale`` (LSTM): the learner's heads are scaled so that its state moves its draws; an agent 1, whose
        state the batch does not record, keeps the fresh model's small heads, so that its draws stay clear of its error."""
        m = self._weights(kind, seed, head_scale)
        self.made.append((m, kind, seed, head_scale))
        return m

    def second(self):
        for m, kind, seed, scale in self.made:
            if kind == "greedy":  # no weights
                continue
            m.load_state_dict(self._weights(kind, seed + 1000, scale).state_dict())


def _population(models):
    """Two network members and a BC member."""
    return [models.make("cnn", 21), models.make("bc", 22), models.make("cnn", 23)]


def build(case, use_graph, seed=7):
    """(rollout, reference spec, models, env, rs) of a case."""
    from overcooked_ai_b200.selfplay import AgentPairRollout, SelfPlayRollout

    env, rs = _env(case, seed)
    n = env.n_envs
    rng = np.random.RandomState(n)
    models = _Models(env)
    kw = dict(use_graph=use_graph, seed=seed, episode_capacity=1 if case["episode_capacity"] == "1" else 3,
              use_phi=case["use_phi"] == "on")
    if case["path"] == "float32":
        kw["autocast_dtype"] = None
    spec = dict(seed=seed, use_phi=kw["use_phi"], capacity=kw["episode_capacity"], seq_len=SEQ_LEN)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.int32)).cuda()
    if case["class"] == "SelfPlayRollout":
        learner = case["learner"]
        if learner in ("cnn", "lstm"):
            model = models.make(learner, 1)
        else:
            model = [models.make("cnn", k + 1) for k in range(3)]
        if learner == "blocks":
            kw["blocks"] = spec["blocks"] = [n // 2, n // 4, n - n // 2 - n // 4]
        elif learner == "pairs":
            pairs = rng.randint(0, 3, size=(n, 2))
            kw["pairs"], spec["pairs"] = dev(pairs), pairs
        elif learner == "pair_weights":
            kw["pair_weights"] = spec["pair_weights"] = PAIR_WEIGHTS
        partner = case["partner"]
        p = None if partner == "none" else models.make(partner, 11) if partner in ("bc", "cnn", "greedy") else _population(models)
        if p is not None:
            kw["partner"] = p
            kw["bc_factor"] = spec["bc_factor"] = BC_FACTOR[case["bc_factor"]]
        if partner == "population_fixed":
            member = rng.randint(0, 3, size=n)
            kw["member"], spec["member"] = dev(member), member
        elif partner == "population_drawn":
            kw["member_weights"] = spec["member_weights"] = WEIGHTS
        kw["reward_shaping_factor"] = spec["factor"] = 0.75
        kw["fused_first_layer"], kw["fused_tail"], kw["fused_wide"] = FUSED[case["path"]]
        kw["max_seq_len"] = SEQ_LEN
        assert set(kw) | {"env", "model"} == passed_arguments(case), sorted(set(kw) ^ passed_arguments(case))
        ro = SelfPlayRollout(env, model=model, **kw)
        spec.update(kind="self_play", learner=model, partner=p)
    else:
        a0 = models.make(case["agent0"], 1)
        a1 = case["agent1"]
        a1 = models.make(a1, 11, head_scale=1.0) if a1 in ("cnn", "bc", "lstm", "greedy") else _population(models)
        if case["agent1"] == "population_fixed":
            member = rng.randint(0, 3, size=n)
            kw["member"], spec["member"] = dev(member), member
        elif case["agent1"] == "population_drawn":
            kw["member_weights"] = spec["member_weights"] = WEIGHTS
        if case["seats"] == "swap":
            swap = rng.randint(0, 2, size=n)
            kw["swap"], spec["swap"] = dev(swap), swap
        elif case["seats"] == "random_seats":
            kw["random_seats"] = spec["random_seats"] = True
        kw["max_seq_len"] = SEQ_LEN
        assert set(kw) | {"env", "agents"} == passed_arguments(case), sorted(set(kw) ^ passed_arguments(case))
        ro = AgentPairRollout(env, (a0, a1), **kw)
        spec.update(kind="pair", agents=(a0, a1), factor=1.0)
    if case["phase"] == "staggered":  # construction kept the timesteps
        assert np.array_equal(_np(env.state[:, 0]), staggered_timesteps(n, case["horizon"])), "phase"
    return ro, spec, models, env, rs


# ---------------------------------------------------------------------------------------------------------- checking
def _np(t):
    return t.detach().cpu().numpy()


def _device_counters(ro, ref):
    """The device's counter for each counter name of the reference."""
    out = {}
    pair = ref.pair_kind
    for name in ref.counters:
        if name == "draw":
            t = ro._draw_counter
        elif name == "seat":
            t = ro._seat_counter
        elif name == "partner":
            t = ro._partner_counter
        elif name == "member_draw":
            t = ro._pop._counter
        elif name == "pair_draw":
            t = ro._learners._counter
        elif name.startswith("member"):
            t = (ro.agents[1] if pair else ro._partner).agents[int(name[6:])]._counter
        else:
            t = ro.agents[int(name[-1])]._counter
        out[name] = int(t[0])
    return out


def _check_live(ro, ref, where):
    env = ro.env
    assert np.array_equal(_np(env.state), ref.state), where
    assert np.array_equal(_np(ro.ret_sparse), ref.ret_sparse), where
    if not ref.pair_kind:
        assert np.array_equal(_np(ro.ret_mixed), ref.ret_mixed), where
    for got, want in zip(ro.stats.state_tensors(), ref.ep.running()):
        assert np.array_equal(_np(got), want), where
    if ref.pair_kind or ref.partner is not None:
        assert np.array_equal(_np(ro.partner_seat), ref.partner_seat), where
    if ro._pop is not None:
        assert np.array_equal(_np(ro.member), ref.member), where
    if getattr(ro, "pair", None) is not None:
        assert np.array_equal(_np(ro.pair), ref.pair), where
    assert _device_counters(ro, ref) == ref.counters, (where, _device_counters(ro, ref), ref.counters)


def _check_records(records, want, where):
    got = records.finished()
    assert set(got) == set(want), (where, sorted(got), sorted(want))
    for k in want:
        assert np.array_equal(_np(got[k]), want[k]), (where, k)


def _lstm_restart(ref, b, t, rows=None):
    """The reference's LSTM learner restarts chunk t // L from the batch's state (one-view: at agent 0's rows)."""
    a = ref.lstm_agent()
    k = t // b.seq_len
    h, c = _np(b.state_h[k].float()).astype(np.float64), _np(b.state_c[k]).astype(np.float64)
    if rows is None:
        a.h[:], a.c[:] = h, c
    else:
        a.h[rows], a.c[rows] = h, c


def _close(got, want, tol=R.REPLAY_TOL):
    return np.abs(np.asarray(got, np.float64) - want) <= tol * (1 + np.abs(want))


def _check_window(ro, ref, b, T, keep_logits, where, live_h=None, bootstrap=False):
    n, pair = ro.env.n_envs, ref.pair_kind
    e = np.arange(n)
    st, ac, dn = _np(b.states), _np(b.actions), _np(b.dones)
    lstm = ref.lstm_agent() is not None
    assert (b.terminal_values is None) == (not bootstrap), where
    ref.begin_window(T, bootstrap)
    outs = []
    for t in range(T):
        p0 = 1 - ref.partner_seat if pair else None
        rows0 = 2 * e + p0 if pair else None
        if lstm and t % b.seq_len == 0:
            # zero state where an episode starts at the chunk; elsewhere at t = 0 the live state the last window left
            started = (dn[t - 1] if t > 0 else ref.prev_done) != 0
            z = np.repeat(started, 2) if not pair else started
            sh = _np(b.state_h[t // b.seq_len].float())
            assert (sh[z] == 0).all(), (where, t)
            if t == 0:
                assert np.array_equal(sh[~z], live_h[~z]), where
            _lstm_restart(ref, b, t, rows0)
        known = np.full(2 * n, -1, np.int64)
        if pair:
            known[rows0] = ac[t]
        else:
            known[:] = ac[t]
        nxt = st[t + 1] if t + 1 < T else _np(ro.env.state)
        o = ref.transition(known, nxt, (p0, _np(b.rewards[t])) if pair else None)
        outs.append(o)
        assert np.array_equal(st[t], o["state"]), (where, t)
    assert np.array_equal(dn, np.stack([o["dones"] for o in outs])), where
    # per-row outputs on the learner's rows
    last = ref.bootstrap()
    # the batch carries a seat, member or pair field exactly where the configuration has one
    assert (b.partner_seat is not None) == (pair or ref.partner is not None), where
    assert (b.partner_member is not None) == ref.ep.members, where
    assert (b.pair is not None) == ref.ep.pairs, where
    if pair:
        rows = np.stack([2 * e + (1 - o["partner_seat"]) for o in outs])          # [T, N] agent 0's joint rows
        pick = lambda key: np.stack([o[key][r] for o, r in zip(outs, rows)])
        want_r = np.stack([o["rewards"].reshape(-1)[r] for o, r in zip(outs, rows)])
        mask = np.ones((T, n), bool)
        assert np.array_equal(_np(b.partner_seat), np.stack([o["partner_seat"] for o in outs])), where
    else:
        pick = lambda key: np.stack([o[key] for o in outs])
        want_r = np.stack([o["rewards"].reshape(-1) for o in outs])
        mask = np.stack([R.learner_mask(o["partner_seat"]) for o in outs]).astype(bool)
        if b.partner_seat is not None:
            assert np.array_equal(_np(b.partner_seat), np.stack([o["partner_seat"] for o in outs])), where
        assert np.array_equal(_np(b.learner_mask).astype(bool), mask), where
        if b.pair is not None:
            assert np.array_equal(_np(b.pair), np.stack([o["pair"] for o in outs])), where
    if b.partner_member is not None:
        assert np.array_equal(_np(b.partner_member), np.stack([o["member"] for o in outs])), where
    assert np.array_equal(ac, pick("actions")), where
    assert np.array_equal(_np(b.rewards), want_r), where
    values, logp, scores = pick("values"), pick("logp"), pick("scores")
    gv, gl = _np(b.values), _np(b.logp)
    if lstm:
        assert _close(gv[mask], values[mask]).all(), (where, np.abs(gv[mask] - values[mask]).max())
        bound = 4 * R.REPLAY_TOL * (1 + np.abs(scores[mask][:, :6]).max(1))
        assert (np.abs(gl[mask] - logp[mask]) <= bound).all(), where
        assert _close(_np(b.last_values), last).all(), where
    else:
        assert np.array_equal(gv[mask], values[mask]), where
        assert (np.abs(gl[mask] - logp[mask]) <= 1e-5 * (1 + np.abs(logp[mask]))).all(), (where, np.abs(gl[mask] - logp[mask]).max())
        assert np.array_equal(_np(b.last_values), last), where
    if keep_logits:
        lg = _np(b.logits)
        if lstm:
            assert _close(lg[mask][:, :6], scores[mask][:, :6]).all(), where
        else:
            assert np.array_equal(lg[mask][:, :6], scores[mask][:, :6]), where
    # GAE on the reference's rewards and dones, and its values (the device's own for the LSTM, whose values are not exact)
    v = np.where(mask, gv if lstm else values, 0).astype(np.float32)
    lv = _np(b.last_values) if lstm else last
    if bootstrap:  # the terminal values on every row, the zeros included; GAE bootstraps from them at each episode end
        tv = pick("terminal_values")
        got = _np(b.terminal_values)
        assert np.array_equal(got.view(np.int32), tv.view(np.int32)), (where, np.argwhere(got != tv)[:8].tolist())
        adv, tgt = gae_horizon_f32(want_r, v, dn, tv, np.asarray(lv, np.float32), GAMMA, LAM)
    else:
        adv, tgt = (R.gae_view_f32 if pair else gae_f32)(want_r, v, dn, lv, GAMMA, LAM)
    assert np.array_equal(_np(b.advantages)[mask], adv[mask]), where
    assert np.array_equal(_np(b.value_targets)[mask], tgt[mask]), where
    _check_records(b.episodes, ref.ep.finished(), where)
    assert np.array_equal(_np(b.episodes.dropped), ref.ep.dropped), where
    ref.end_window()
    return outs


def _certify(ref, case, states=None):
    """The exactness premise on this path: every accumulation of every exact network, with its current weights, is
    certified on the reference's current states (or ``states``: the window's terminal records), with operands of at most
    8 significant bits (bf16; TF32 keeps 11, float32 24).  ``P.exact_cnn`` bounds every unit over all encodings; this
    checks that claim where it is relied on."""
    states = ref.state if states is None else states
    if len(states) == 0:
        return
    obs = cpu.encode_lossless(ref.host.tables, states, ref.host.W, ref.host.H, ref.host.horizon)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    for a in ref.agents():
        if a.kind != "cnn":
            continue
        certs, bits = R.cnn_certificates(a.model, obs)
        assert all(c.holds() for c in certs) and bits <= 8, ("premise", case, bits, "allow_tf32=%s" % tf32)


def _setters(ro, ref, case):
    ro.reward_shaping_factor = 0.5
    ref.factor = 0.5
    if case.get("bc_factor") is not None:
        ro.bc_factor = ref.bc = BC_FACTOR_LATER[case["bc_factor"]]
    if "population_drawn" in (case.get("partner"), case.get("agent1")):
        ro.member_weights = WEIGHTS_LATER
        ref.set_member_weights(WEIGHTS_LATER)
    if case.get("learner") == "pair_weights":
        ro.pair_weights = PAIR_WEIGHTS_LATER
        ref.set_pair_weights(PAIR_WEIGHTS_LATER)


# ---------------------------------------------------------------------------------------------------------- the path
def _launched(fn):
    from test_gpu_env_forms import _launched as launched
    return launched(fn)


def _library(names):
    return any(re.search(r"gemm|nvjet|cutlass|xmma|sm90_|sm80_", k.lower()) for k in names if not k.startswith("ovc::"))


def _check_path(case, models, names):
    has = lambda prefix: any(k.startswith(prefix) for k in names)
    kinds = {made[1] for made in models.made}
    path = case["path"]
    k2, k7, k9 = has("ovc::encode_kernel"), has("ovc::encode_linear"), has("ovc::wide_layers")
    k8, draw, k11, lib = has("ovc::policy_tail"), has("ovc::sample_actions"), has("ovc::lstm_head"), _library(names)
    nets = kinds & {"cnn", "lstm"}
    want = {
        "k7_k9_k8": dict(k2=False, k7=True, k9=True, k8=True, draw=False, lib=False),
        "learner_rows": dict(k2=False, k7=True, k9=True, k8=True, draw=False, lib=False),
        "k7_library_draw": dict(k2=False, k7=True, k9=False, k8=False, lib=True),
        "k2_library_k8": dict(k2=True, k7=False, k9=False, k8=True, draw=False, lib=True),
        "k2_library_draw": dict(k2=True, k7=False, k9=False, k8=False, lib=True),
        "float32": dict(k2=True, k7=False, k9=False, k8=False, lib=True),
    }[path]
    got = dict(k2=k2, k7=k7, k9=k9, k8=k8, draw=draw, lib=lib)
    for k, v in want.items():
        assert got[k] == v, (case, k, sorted(names))
    if path in ("k7_library_draw", "k2_library_draw", "float32") and "cnn" in nets:
        assert draw, (case, sorted(names))
    assert k11 == ("lstm" in nets), (case, sorted(names))
    if path == "learner_rows":
        assert has("ovc::learner_rows_kernel") and has("ovc::encode_linear_masked"), (case, sorted(names))
    assert has("ovc::partner_policy") == ("bc" in kinds), (case, sorted(names))
    assert has("ovc::greedy_actions_kernel") == ("greedy" in kinds), (case, sorted(names))


def _check_window_path(case, names):
    """The kernels of the first eager collect() window: with bootstrap_horizon, the compaction (ovc_horizon_rows) and K7's
    rows form exactly where the learner runs K7 -> K9 -> K8 (a network partner's members run the rows form too), and the
    horizon GAE in the batch's form (two views, or agent 0's one) in place of the plain GAE kernel."""
    has = lambda prefix: any(k.startswith(prefix) for k in names)
    on = case["bootstrap_horizon"] == "on"
    fused = case["path"] in ("k7_k9_k8", "learner_rows")
    rows_form = any(re.fullmatch(r"ovc::encode_linear_kernel<\d+,1,1>", k) for k in names)
    assert has("ovc::horizon_rows_kernel") == (on and fused), (case, sorted(names))
    if case.get("partner", case.get("agent1")) in ("cnn", "population_fixed", "population_drawn"):
        assert rows_form or not (on and fused), (case, sorted(names))
    else:
        assert rows_form == (on and fused), (case, sorted(names))
    form = "float" if case["class"] == "AgentPairRollout" else "float2"
    horizon_gae = {k for k in names if k.startswith("ovc::gae_horizon_kernel")}
    assert horizon_gae == ({"ovc::gae_horizon_kernel<%s>" % form} if on else set()), (case, sorted(names))
    assert has("ovc::gae_kernel<") == (not on), (case, sorted(names))


# ---------------------------------------------------------------------------------------------------------- the test
# The share of LSTM draws whose top-2 Gumbel gap is within 2 REPLAY_TOL (1 + max |logit|), so checked only as one of the
# tied actions: 3 - 4 % on these models and grids; a larger bound would silently stop checking the LSTM's draws.
LSTM_OPEN_MAX = 0.08


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", sorted(CONFIGURATIONS))
def test_rollout_form_vs_reference(name, use_graph):
    case = CONFIGURATIONS[name]
    ro, spec, models, env, rs = build(case, use_graph)
    ref = R.RolloutReference(_host(env, rs, spec["use_phi"]), _np(env.state), spec)
    certify = (lambda: None) if use_graph else (lambda: _certify(ref, name))  # the graph run reaches the same states
    certify()
    _check_live(ro, ref, "construction")
    T = case["T"]
    bootstrap = case["bootstrap_horizon"] == "on"
    collect_agent0 = case.get("agent0") not in SCRIPTED
    if collect_agent0:
        for w in range(2):
            if w == 1:
                _setters(ro, ref, case)
                models.second()
                ro.sync_weights()
                ref.sync()
                certify()  # the second weights, on the states the first window reached
            lstm = ref.lstm_agent()
            live_h = None if lstm is None else _np((ro.h if not ref.pair_kind else ro.agents[0].h).float()).copy()
            collect = lambda: ro.collect(T, GAMMA, LAM, keep_logits=w == 1, bootstrap_horizon=bootstrap)
            if w == 0 and not use_graph:  # the kernels of the first eager window
                got = []
                _check_window_path(case, _launched(lambda: got.append(collect())))
                b = got[0]
            else:
                b = collect()
            _check_window(ro, ref, b, T, w == 1, (name, "window", w), live_h, bootstrap)
            if bootstrap and not use_graph:  # the terminal values are exact only where the premise holds on their records
                _certify(ref, name, np.concatenate(ref.terminal_records))
            _check_live(ro, ref, (name, "after window", w))
    else:  # a BC or greedy agent 0 has no learner: run() only
        _setters(ro, ref, case)
    certify()
    ref.begin_run()

    def run():
        for t in range(T):
            ro.run(1)
            o = ref.transition(_np(ro.actions).reshape(-1))
            assert np.array_equal(_np(ro.actions).reshape(-1), o["actions"]), (name, "run", t)
    if use_graph:
        run()
    else:  # the kernels of the eager transitions are the path's
        _check_path(case, models, _launched(run))
    ref.end_run()
    _check_live(ro, ref, (name, "after run"))
    ref.begin_run()
    _check_records(ro.episodes, ref.ep.finished(), (name, "run records"))
    assert np.array_equal(_np(ro.episodes.dropped), ref.ep.dropped), name
    ref.end_run()
    assert ref.ties <= 0.005 * ref.draws, (ref.ties, ref.draws)
    # an LSTM draw within the heads' error bound is checked only as one of the tied actions: most must be clear
    assert ref.lstm_open <= LSTM_OPEN_MAX * ref.lstm_draws, (ref.lstm_open, ref.lstm_draws)
    print("%s: %d near-ties in %d draws; %d of %d LSTM draws within the error bound"
          % (name, ref.ties, ref.draws, ref.lstm_open, ref.lstm_draws))
