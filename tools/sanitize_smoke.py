#!/usr/bin/env python
"""Every kernel family at smoke sizes, for compute-sanitizer (memcheck / racecheck / synccheck / initcheck):
K1 with each record-I/O strategy (2-D TMA tile, 1-D bulk TMA, direct), K5 (the rollout kernel, int32 and
host-transfer formats, standard and random-start auto-resets, 16- / 32- / 64-word records, a partial last tile),
the round-1 fused path, K4 reset (copy + random), K2, K3, K6, the host-buffer pipeline, the policy kernels K7 / K8 and
the sample-batch kernels (logp draws, ovc_record_transition, ovc_gae through SelfPlayRollout.collect), K10 and the seat draw,
the episode statistics of ovc_record_transition_stats, the LSTM policy (K8's hidden output, K11), and agent pairs (the
one-view forms of K7, K8, K11 and the draw).  Results are checked
against the CPU oracle on the way, so a run under the sanitizer is also a parity run.

    compute-sanitizer --tool racecheck python tools/sanitize_smoke.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

from oracle import cpu  # noqa: E402
from overcooked_ai_b200 import _native, wire  # noqa: E402
from overcooked_ai_b200.batched import BatchedOvercookedEnv, HostRolloutPipeline  # noqa: E402

rng = np.random.RandomState(0)


def acts_for(T, n):
    a = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32)
    a[rng.rand(T, n, 2) < 0.3] = 5
    return a


def check(env, acts, split, rs=None):
    ref_state = env.state.cpu().numpy().copy()
    ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=env.horizon, flags=int(env.auto_reset), n_threads=2, rs=rs)
    d = torch.from_numpy(acts).cuda()
    for t in range(split):
        out = env.step(d[t])
        for g, w in zip(out, ref):
            assert np.array_equal(g.cpu().numpy(), w[t])
    out = env.rollout(d[split:].contiguous())
    for g, w in zip(out, ref):
        assert np.array_equal(g.cpu().numpy(), w[split:])
    assert np.array_equal(env.state.cpu().numpy(), ref_state)


n = 333  # partial last tile for every tile size
for io in (_native.IO_TMA_TENSOR, _native.IO_TMA_BULK, _native.IO_DIRECT):
    env = BatchedOvercookedEnv(["cramped_room"], n, horizon=25, io=io, auto_reset=True)
    check(env, acts_for(40, n), 8)
print("K1 x3 I/O strategies + K5 (S=16) ok", flush=True)
env = BatchedOvercookedEnv(["cramped_room", "counter_circuit", "asymmetric_advantages"], n, horizon=30, auto_reset=True)
check(env, acts_for(70, n), 5)
env = BatchedOvercookedEnv(["cramped_room", "counter_circuit"], n, horizon=30, auto_reset=False)
check(env, acts_for(50, n), 5)
print("K5 mixed layouts (S=32), with and without auto-reset ok", flush=True)
env = BatchedOvercookedEnv(["marshmallow_experiment"], 100, horizon=30, auto_reset=True)
check(env, acts_for(45, 100), 3)
print("K5 S=64 ok", flush=True)
env = BatchedOvercookedEnv(["cramped_room", "coordination_ring"], n, horizon=20, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=9)
rs = cpu.random_start(9, 0.6, True)
ref = env.state.cpu().numpy().copy()
cpu.reset_random(env._tab_host, env._starts_host, ref, rs, env_layout=env.env_layout_host)
ref[:, 3] = env.state.cpu().numpy()[:, 3]
check(env, acts_for(50, n), 4, rs=rs)
print("K4 random reset + K5 random-start auto-reset ok", flush=True)
# host-transfer formats through K5 and the native pipeline
env = BatchedOvercookedEnv(["cramped_room", "counter_circuit"], n, horizon=30, auto_reset=True)
a = acts_for(48, n)
ref_state = env.state.cpu().numpy().copy()
ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, a, horizon=30, flags=1, n_threads=2)
for kw in ({"codes": True}, {"packed": True}, {"narrow": True}, {}):
    env.reset()
    pipe = HostRolloutPipeline(env, 48, chunk=16, **kw)
    ha = torch.from_numpy(wire.pack_actions(a)).pin_memory() if kw.get("codes") else torch.from_numpy(a.astype(np.uint8) if kw else a).pin_memory()
    out = pipe.run(ha)
    torch.cuda.synchronize()
    if kw.get("codes"):
        dense = env.expand_codes(out[3], events=True)
        for k, w in zip(("sparse", "shaped", "done", "events"), ref):
            assert np.array_equal(dense[k].numpy(), w)
    else:
        assert np.array_equal(out[0].numpy().astype(np.int32), ref[0])
    assert np.array_equal(env.state.cpu().numpy(), ref_state)
    pipe.close()
print("host-buffer pipeline, 4 transfer formats ok", flush=True)
# round-1 fused path (step_kernel with n_steps > 1) stays reachable: more than 8 layouts keep the tables in global memory
names = ["cramped_room", "coordination_ring", "forced_coordination", "five_by_five", "centre_pots", "centre_objects", "bottleneck",
         "simple_o", "scenario2", "scenario3"]
env = BatchedOvercookedEnv(names, n, horizon=30, auto_reset=True)
check(env, acts_for(40, n), 3)
print("fused step_kernel path (global tables) ok", flush=True)
# observation kernels
env = BatchedOvercookedEnv(["cramped_room"], n, horizon=400, auto_reset=True)
env.rollout(torch.from_numpy(acts_for(120, n)).cuda())
st = env.state.cpu().numpy()
for dt in (torch.float32, torch.uint8, torch.bfloat16, torch.int32):
    enc = env.lossless_state_encoding(dtype=dt)
    want = cpu.encode_lossless(env._tab_host, st, 5, 4, horizon=400)
    assert np.array_equal(enc.float().cpu().numpy(), want.astype(np.float32))
feat = env.featurize_state(num_pots=2).cpu().numpy()
lut = np.stack([l.feature_lut() for l in env.layouts]).view(np.uint8).reshape(1, -1)
assert np.array_equal(feat.astype(np.float64), cpu.featurize(env._tab_host, lut, st, 2))
phi = env.potential(0.99).cpu().numpy()
assert phi.shape == (n,)
env.reset(torch.from_numpy((rng.rand(n) < 0.5).astype(np.int32)).cuda())
torch.cuda.synchronize()
print("K2 x4 dtypes, K3, K6, K4 masked reset ok", flush=True)
# K7 (first policy layer from the record), K8 (dense tail + draw), the draw / return kernels, and the self-play transition on them
from overcooked_ai_b200.selfplay import SelfPlayRollout  # noqa: E402

env = BatchedOvercookedEnv(["cramped_room"], n, horizon=40, auto_reset=True)
env.rollout(torch.from_numpy(acts_for(25, n)).cuda())
wt = ((torch.rand((520, 128), device="cuda") - 0.5) * 0.1).to(torch.bfloat16)
bias = (torch.rand(128, device="cuda") - 0.5) * 0.2
obs = env.lossless_state_encoding(dtype=torch.float32).view(2 * n, 520)
want = torch.nn.functional.leaky_relu(obs @ wt.float() + bias, 0.2)
got = env.encoded_linear(wt, bias, neg_slope=0.2).float()
assert ((got - want).abs() <= want.abs() * 2.0 ** -8 + 1e-4).all()  # bf16 output of a float32 accumulation
sp = SelfPlayRollout(env, use_graph=False, seed=3)
assert sp.fused_first_layer and sp.fused_tail
ref_state = env.state.cpu().numpy().copy()
for t in range(6):
    sp.run(1)
    cpu.step(env._tab_host, env._starts_host, ref_state, sp.actions.cpu().numpy(), horizon=40, flags=1)
    assert np.array_equal(env.state.cpu().numpy(), ref_state)
sp2 = SelfPlayRollout(env, model=sp.model, use_graph=False, fused_tail=False)
sp2.run(3)
torch.cuda.synchronize()
print("K7, K8, sample / accumulate kernels, self-play transitions ok", flush=True)
# sample batches: K8 and the draw kernel with logp, ovc_record_transition and ovc_gae, through collect()
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
from ppo_reference import gae_f32, log_softmax_at  # noqa: E402

for r in (sp, sp2):
    r.reward_shaping_factor = 0.5
    ref_state = env.state.cpu().numpy().copy()
    b = r.collect(12, 0.99, 0.95, keep_logits=True)
    st, ac, rw, dn = (x.cpu().numpy() for x in (b.states, b.actions, b.rewards, b.dones))
    for t in range(12):
        assert np.array_equal(st[t], ref_state)
        sp_, sh_, d_, _ = cpu.step(env._tab_host, env._starts_host, ref_state, ac[t].reshape(n, 2), horizon=40, flags=1)
        assert np.array_equal(rw[t].reshape(n, 2), sp_[:, None].astype(np.float32) + np.float32(0.5) * sh_.astype(np.float32))
        assert np.array_equal(dn[t], (d_ != 0).astype(np.uint8))
        lp = log_softmax_at(b.logits[t].cpu().numpy(), ac[t], 6)
        assert (np.abs(b.logp[t].cpu().numpy() - lp) <= 1e-5 * (1 + np.abs(lp))).all()
    adv, tgt = gae_f32(rw, b.values.cpu().numpy(), dn, b.last_values.cpu().numpy(), 0.99, 0.95)
    assert np.array_equal(b.advantages.cpu().numpy(), adv) and np.array_equal(b.value_targets.cpu().numpy(), tgt)
torch.cuda.synchronize()
print("K8 / draw with logp, record_transition, GAE through collect() ok", flush=True)
# the BC partner: K10 (featurize_state + MLP + draw) and the seat draw, alone and through collect()
from overcooked_ai_b200.selfplay import BCPolicy  # noqa: E402

bc = BCPolicy().cuda()
seat = torch.from_numpy(rng.randint(-1, 2, size=n).astype(np.int32)).cuda()
acts = torch.full((n, 2), 9, dtype=torch.int32, device="cuda")
scores = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
env.partner_actions(bc.tables(), seat, torch.zeros(2, dtype=torch.int64, device="cuda"), seed=5, out=acts, scores=scores)
sh = seat.cpu().numpy()
a_np = acts.cpu().numpy()
assert (a_np[sh >= 0, sh[sh >= 0]] < 6).all() and (a_np[sh < 0] == 9).all()
feat = env.featurize_state(num_pots=2)[torch.arange(n, device="cuda"), seat.clamp(min=0).long()]
want = bc(feat)
assert ((scores[seat >= 0, :6] - want[seat >= 0]).abs() <= 0.05 * (1 + want[seat >= 0].abs())).all()  # bf16 operands
factor = torch.full((1,), 0.5, dtype=torch.float32, device="cuda")
env.assign_partners(seat, factor, torch.zeros(2, dtype=torch.int64, device="cuda"), seed=6, done=env.done)
sp3 = SelfPlayRollout(env, model=sp.model, use_graph=False, seed=3, partner=bc, bc_factor=0.5)
b = sp3.collect(12, 0.99, 0.95)
assert b.learner_mask.shape == (12, 2 * n) and int(b.learner_mask.sum()) >= 12 * n
# three 5x4 layouts interleaved env by env: K10, K7 and the statistics index their per-layout tables with ids 0..2 in one tile
envp = BatchedOvercookedEnv(["cramped_room", "mdp_test", "bonus_order_test"], n, horizon=6, auto_reset=True,
                            env_layout=np.arange(n) % 3, rnd_obj_prob_thresh=0.6, seed=4)
envp.rollout(torch.from_numpy(acts_for(9, n)).cuda())
st = envp.state.cpu().numpy().copy()
scores.fill_(float("nan"))
envp.partner_actions(bc.tables(), seat, torch.zeros(2, dtype=torch.int64, device="cuda"), seed=5, scores=scores)
feat = envp.featurize_state(num_pots=2)
assert np.array_equal(feat.cpu().numpy().astype(np.float64), cpu.featurize(envp._tab_host, envp.feature_lut().cpu().numpy(), st, 2))
want = bc(feat[torch.arange(n, device="cuda"), seat.clamp(min=0).long()])
assert ((scores[seat >= 0, :6] - want[seat >= 0]).abs() <= 0.05 * (1 + want[seat >= 0].abs())).all()  # bf16 operands
sp4 = SelfPlayRollout(envp, model=sp.model, use_graph=False, seed=3, partner=bc, bc_factor=0.5)
assert sp4.fused_first_layer and sp4.fused_wide and sp4.fused_tail
b = sp4.collect(1, 0.99, 0.95)
cpu.step(envp._tab_host, envp._starts_host, st, b.actions[0].cpu().numpy().reshape(n, 2), horizon=6, flags=1, rs=cpu.random_start(4, 0.6))
assert np.array_equal(envp.state.cpu().numpy(), st)
torch.cuda.synchronize()
print("K10 partner policy, assign_partners, collect() with a partner, on one layout and on three interleaved ok", flush=True)
# the episode statistics (ovc_record_transition_stats): horizon 5 over 15 transitions into 2 slots (the third episode is
# dropped), random starts so that episodes deliver, against the numpy restatement
from episode_reference import EpisodeReference, rewards_f32  # noqa: E402
from overcooked_ai_b200.batched import EpisodeRecords, EpisodeStats  # noqa: E402

env6 = BatchedOvercookedEnv(["cramped_room", "coordination_ring"], n, horizon=5, auto_reset=True, rnd_obj_prob_thresh=0.6, seed=2)
rs6 = cpu.random_start(2, 0.6)
ref_state = env6.state.cpu().numpy().copy()
stats, recs = EpisodeStats(env6), EpisodeRecords(env6, 2)
ref = EpisodeReference(np.stack([l.deliver_value for l in env6.layouts]), ref_state[:, 3] & 0xFF, 2)
for a in acts_for(15, n):
    env6.step(torch.from_numpy(a).cuda())
    env6.record_transition(factor, stats=stats, records=recs, partner_seat=seat)
    sp_, sh_, d_, ev_ = cpu.step(env6._tab_host, env6._starts_host, ref_state, a, horizon=5, flags=1, rs=rs6)
    ref.step(sh_, d_, ev_, ref_state[:, 3] & 0xFF, rewards_f32(sp_, sh_, 0.5), seat.cpu().numpy())
fin = recs.finished()
for k, want in ref.finished().items():
    assert np.array_equal(fin[k].cpu().numpy(), want), k
assert (recs.dropped.cpu().numpy() == ref.dropped).all() and (ref.dropped == 1).all()
torch.cuda.synchronize()
print("episode statistics (record_transition with stats) ok", flush=True)
# the LSTM policy: K8's hidden output and K11 (ovc_lstm_head) through collect() on a 5x4 grid (K7 -> K9 -> K8 hidden -> K11)
# and on a 9x5 grid (library layers -> K11), episodes ending inside the window
from overcooked_ai_b200.selfplay import RllibLSTMShapedCNN  # noqa: E402

for name in ("cramped_room", "asymmetric_advantages"):
    env7 = BatchedOvercookedEnv(name, 37, horizon=3, auto_reset=True)
    l7 = env7.layouts[0]
    sp7 = SelfPlayRollout(env7, model=RllibLSTMShapedCNN(l7.width, l7.height), use_graph=False, seed=4, max_seq_len=2)
    st = env7.state.cpu().numpy().copy()
    b = sp7.collect(5, 0.99, 0.95, keep_logits=True)
    for t in range(5):
        cpu.step(env7._tab_host, env7._starts_host, st, b.actions[t].cpu().numpy().reshape(-1, 2), horizon=3, flags=1)
    assert np.array_equal(env7.state.cpu().numpy(), st) and b.dones.any()
torch.cuda.synchronize()
print("LSTM policy (K8 hidden output, K11) through collect() ok", flush=True)
# agent pairs: the one-view forms of K7 -> K9 -> K8, K8 hidden -> K11 and K10 on a 5x4 grid, and the library layers with
# the one-view draw on a 9x5 grid, mixed seats, episodes ending inside the run; the environments follow the oracle
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN  # noqa: E402

for name, agents in (("cramped_room", lambda W, H: (RllibShapedCNN(W, H), RllibLSTMShapedCNN(W, H))),
                     ("cramped_room", lambda W, H: (RllibLSTMShapedCNN(W, H), BCPolicy())),
                     ("asymmetric_advantages", lambda W, H: (RllibShapedCNN(W, H), RllibLSTMShapedCNN(W, H)))):
    env8 = BatchedOvercookedEnv(name, 37, horizon=3, auto_reset=True)
    l8 = env8.layouts[0]
    swap8 = torch.from_numpy((rng.rand(37) < 0.5).astype(np.int32)).cuda()
    pair = AgentPairRollout(env8, agents(l8.width, l8.height), swap=swap8, seed=4, use_graph=False)
    st = env8.state.cpu().numpy().copy()
    for t in range(5):
        pair.run(1)
        cpu.step(env8._tab_host, env8._starts_host, st, pair.actions.cpu().numpy(), horizon=3, flags=1)
    assert np.array_equal(env8.state.cpu().numpy(), st)
torch.cuda.synchronize()
print("agent pairs (one-view K7 / K8 / K11 / draw, K10) ok", flush=True)
# a learner next to a fixed partner: collect() with random seats (the learner-row record kernel with statistics, the seat
# draw, the learner-row GAE) on a 5x4 grid (CNN and LSTM learners) and on a 9x5 grid (library layers), 37 environments,
# episodes ending inside the window
for name, agents in (("cramped_room", lambda W, H: (RllibShapedCNN(W, H), BCPolicy())),
                     ("cramped_room", lambda W, H: (RllibLSTMShapedCNN(W, H), RllibShapedCNN(W, H))),
                     ("asymmetric_advantages", lambda W, H: (RllibShapedCNN(W, H), RllibShapedCNN(W, H)))):
    env9 = BatchedOvercookedEnv(name, 37, horizon=3, auto_reset=True)
    l9 = env9.layouts[0]
    pair = AgentPairRollout(env9, agents(l9.width, l9.height), seed=4, use_graph=False, random_seats=True, max_seq_len=2)
    b = pair.collect(5, 0.99, 0.95, keep_logits=True)
    assert b.dones.any() and (b.partner_seat >= 0).all()
torch.cuda.synchronize()
print("learner-row collect (record_transition_view, gae_view, seat draw) ok", flush=True)
# a population of partners: ovc_group_members, ovc_assign_members and the rows forms of K7 / K9 / K8 next to K10 on a 5x4
# grid, the library layers with the rows form of the draw on a 9x5 grid, members drawn per episode (one of weight 0) and
# fixed; the environments follow the oracle
for name, fixed in (("cramped_room", False), ("asymmetric_advantages", False), ("cramped_room", True)):
    env10 = BatchedOvercookedEnv(name, 37, horizon=3, auto_reset=True)
    l10 = env10.layouts[0]
    W, H = l10.width, l10.height
    kw = dict(member=torch.from_numpy(rng.randint(0, 3, 37).astype(np.int32)).cuda()) if fixed else dict(member_weights=[1.0, 0.0, 2.0])
    pop = AgentPairRollout(env10, (RllibShapedCNN(W, H), [RllibShapedCNN(W, H), RllibShapedCNN(W, H), BCPolicy()]), seed=4,
                           use_graph=False, random_seats=True, episode_capacity=2, **kw)
    st = env10.state.cpu().numpy().copy()
    for t in range(5):
        pop.run(1)
        cpu.step(env10._tab_host, env10._starts_host, st, pop.actions.cpu().numpy(), horizon=3, flags=1)
    assert np.array_equal(env10.state.cpu().numpy(), st)
    b = pop.collect(5, 0.99, 0.95)
    assert b.dones.any() and len(b.episodes.finished()["partner_member"]) > 0
torch.cuda.synchronize()
print("population (group / assign members, rows forms of K7 / K9 / K8 and the draw, K10) ok", flush=True)
# self-play mixtures: ovc_learner_rows, the masked K7, K9 on the compact rows and the joint K8 for the learner, the rows forms
# for a network partner and a population (a BC member among them) on the paired environments only, on a 5x4 and a 9x5 grid
for name, partner in (("cramped_room", lambda W, H: RllibShapedCNN(W, H)), ("cramped_room", lambda W, H: [RllibShapedCNN(W, H), BCPolicy()]),
                      ("asymmetric_advantages", lambda W, H: [RllibShapedCNN(W, H), BCPolicy()])):
    env11 = BatchedOvercookedEnv(name, 37, horizon=3, auto_reset=True)
    l11 = env11.layouts[0]
    W, H = l11.width, l11.height
    mix = SelfPlayRollout(env11, RllibShapedCNN(W, H), seed=4, use_graph=False, partner=partner(W, H), bc_factor=0.5, episode_capacity=2)
    st = env11.state.cpu().numpy().copy()
    for t in range(5):
        mix.run(1)
        cpu.step(env11._tab_host, env11._starts_host, st, mix.actions.cpu().numpy(), horizon=3, flags=1)
    assert np.array_equal(env11.state.cpu().numpy(), st)
    b = mix.collect(5, 0.99, 0.95)
    assert b.dones.any() and (b.partner_seat == -1).any() and (b.partner_seat >= 0).any()
torch.cuda.synchronize()
print("self-play mixtures (learner rows, masked K7, joint K8, partner rows forms) ok", flush=True)
# use_phi: K6 before K1, K1 without the auto-reset, ovc_potential_shaping (standard and random starts), both forms of
# ovc_record_transition_dense with the episode statistics
for kw in ({}, dict(random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=3)):
    env12 = BatchedOvercookedEnv("cramped_room", 37, horizon=3, auto_reset=True, **kw)
    phi = SelfPlayRollout(env12, RllibShapedCNN(5, 4), seed=4, use_graph=False, use_phi=True, episode_capacity=2)
    st = env12.state.cpu().numpy().copy()
    for t in range(5):
        phi.run(1)
        cpu.step(env12._tab_host, env12._starts_host, st, phi.actions.cpu().numpy(), horizon=3, flags=1,
                 rs=cpu.random_start(3, 0.5, True) if kw else None)
    assert np.array_equal(env12.state.cpu().numpy(), st)
    assert phi.collect(5, 0.99, 0.95).dones.any()
    pair = AgentPairRollout(env12, (RllibShapedCNN(5, 4), BCPolicy()), seed=4, use_graph=False, random_seats=True, use_phi=True)
    assert pair.collect(5, 0.99, 0.95).dones.any()
torch.cuda.synchronize()
print("use_phi (K6, K1 without auto-reset, potential shaping, dense record) ok", flush=True)
print("sanitize_smoke: all ok")
