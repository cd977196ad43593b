"""PPO collection for a learner next to a fixed partner (AgentPairRollout.collect) on the device: the learner-row record and
GAE kernels bit for bit against their two-row forms, the per-episode seats against PPO_BC's seat draw, and whole windows
against SelfPlayRollout (a pair of one model) and PPO_BC (a BC partner) gathered at the learner's rows 2 e + p_t(e)."""
import copy

import numpy as np
import pytest
import torch

import policy_reference as P
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeRecords, EpisodeStats
from overcooked_ai_b200.selfplay import (PARTNER_SEAT_SALT, AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN,
                                         SelfPlayRollout)
from rollout_reference import gae_view_f32
from test_gpu_agent_pair import _exact_wide
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GUARD = 64
GAMMA, LAM = 0.99, 0.95


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _guarded(n, dt, fill):
    """(the first n entries, the whole buffer) of a buffer whose tail of GUARD entries holds ``fill``."""
    full = torch.full((n + GUARD,), fill, dtype=dt, device="cuda")
    return full[:n], full


# ------------------------------------------------------------------------------------------------ the record kernel


@pytest.mark.parametrize("stats", [False, True], ids=["plain", "stats"])
def test_record_view_equals_two_view_rows(stats):
    """Every swap pattern and seat, a fractional factor, N not a multiple of 256, episodes ending on the way: the learner's
    reward equals the two-view reward at row 2 e + p(e); dones, returns, statistics and records equal the two-view call's."""
    rng = np.random.RandomState(4)
    n, horizon, T = 333, 9, 20
    swaps = {"none": None, "zeros": torch.zeros(n, dtype=torch.int32, device="cuda"),
             "ones": torch.ones(n, dtype=torch.int32, device="cuda"), "mixed": _dev(rng.randint(0, 3, n), torch.int32)}
    factor = torch.full((1,), 0.37, dtype=torch.float32, device="cuda")
    for name, swap in swaps.items():
        for seat in (0, 1):
            env = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True, rnd_obj_prob_thresh=0.5, seed=seat)
            p = torch.full((n,), seat, device="cuda") if swap is None else seat ^ (swap != 0).long()
            ps = _dev(rng.randint(0, 2, n), torch.int32)
            two = dict(rewards=torch.empty(2 * n, device="cuda"), dones=torch.empty(n, dtype=torch.uint8, device="cuda"),
                       ret_sparse=torch.zeros(n, dtype=torch.int64, device="cuda"), ret_mixed=torch.zeros(n, device="cuda"))
            one = dict(ret_sparse=torch.zeros(n, dtype=torch.int64, device="cuda"), ret_mixed=torch.zeros(n, device="cuda"))
            one["rewards"], r_full = _guarded(n, torch.float32, float("nan"))
            one["dones"], d_full = _guarded(n, torch.uint8, 7)
            if stats:
                for kw in (two, one):
                    kw.update(stats=EpisodeStats(env), records=EpisodeRecords(env, 3), partner_seat=ps)
            for t in range(T):
                env.step(_dev(rng.randint(0, 6, size=(n, 2)), torch.int32))
                env.record_transition(factor, **two)
                env.record_transition_view(factor, seat, swap, **one)
                want = two["rewards"].view(n, 2)[torch.arange(n, device="cuda"), p]
                assert torch.equal(one["rewards"], want), (name, seat, t)
                for k in ("dones", "ret_sparse", "ret_mixed"):
                    assert torch.equal(one[k], two[k]), (name, seat, t, k)
                assert torch.isnan(r_full[n:]).all() and (d_full[n:] == 7).all()
            if stats:
                for a, b in zip(one["stats"].state_tensors(), two["stats"].state_tensors()):
                    assert torch.equal(a, b), (name, seat)
                for a, b in zip(one["records"].tensors(), two["records"].tensors()):
                    assert torch.equal(a, b), (name, seat)
                assert int(one["records"].count.sum()) >= n


# ------------------------------------------------------------------------------------------------ the GAE kernel


@pytest.mark.parametrize("T", [1, 15, 16, 17, 400])
def test_gae_view_equals_the_float32_loop_and_the_two_row_kernel(T):
    n = 301
    rng = np.random.RandomState(T)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    r = rng.uniform(-2, 5, size=(T, n)).astype(np.float32)
    v = rng.uniform(-3, 3, size=(T, n)).astype(np.float32)
    d = (rng.rand(T, n) < 0.1).astype(np.uint8)
    last = rng.uniform(-3, 3, size=n).astype(np.float32)
    adv, adv_full = _guarded(T * n, torch.float32, float("nan"))
    tgt, tgt_full = _guarded(T * n, torch.float32, float("nan"))
    env.gae_view(_dev(r, torch.float32), _dev(v, torch.float32), _dev(d, torch.uint8), _dev(last, torch.float32), GAMMA, LAM,
                 adv.view(T, n), tgt.view(T, n))
    want_a, want_t = gae_view_f32(r, v, d, last, GAMMA, LAM)
    assert np.array_equal(_np(adv).reshape(T, n).view(np.int32), want_a.view(np.int32))
    assert np.array_equal(_np(tgt).reshape(T, n).view(np.int32), want_t.view(np.int32))
    assert torch.isnan(adv_full[T * n:]).all() and torch.isnan(tgt_full[T * n:]).all()
    # ovc_gae on a two-row layout with the learner at row 2 e + p(e) and other numbers on the other row
    p = rng.randint(0, 2, n)
    r2 = rng.uniform(-2, 5, size=(T, n, 2)).astype(np.float32)
    v2 = rng.uniform(-3, 3, size=(T, n, 2)).astype(np.float32)
    l2 = rng.uniform(-3, 3, size=(n, 2)).astype(np.float32)
    ar = np.arange(n)
    r2[:, ar, p], v2[:, ar, p], l2[ar, p] = r, v, last
    a2, t2 = env.gae(_dev(r2.reshape(T, 2 * n), torch.float32), _dev(v2.reshape(T, 2 * n), torch.float32), _dev(d, torch.uint8),
                     _dev(l2.reshape(-1), torch.float32), GAMMA, LAM)
    assert np.array_equal(_np(a2).reshape(T, n, 2)[:, ar, p].view(np.int32), _np(adv).reshape(T, n).view(np.int32))
    assert np.array_equal(_np(t2).reshape(T, n, 2)[:, ar, p].view(np.int32), _np(tgt).reshape(T, n).view(np.int32))


# ------------------------------------------------------------------------------------------------ seats


def test_random_seats_follow_the_seat_draw_and_change_only_at_episode_ends():
    n, seed = 700, 13
    env = BatchedOvercookedEnv("cramped_room", n, horizon=11, auto_reset=True)
    pair = AgentPairRollout(env, (RllibShapedCNN(5, 4), BCPolicy()), seed=seed, random_seats=True)
    shadow = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    one, counter = torch.ones(1, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
    env.assign_partners(shadow, one, counter, seed=seed ^ PARTNER_SEAT_SALT)
    assert torch.equal(pair.partner_seat, shadow)
    assert 0 < int(shadow.sum()) < n and bool(((shadow == 0) | (shadow == 1)).all())
    for t in range(30):
        before = pair.partner_seat.clone()
        pair.run(1)
        env.assign_partners(shadow, one, counter, seed=seed ^ PARTNER_SEAT_SALT, done=env.done)
        assert torch.equal(pair.partner_seat, shadow), t
        kept = env.done == 0
        assert torch.equal(pair.partner_seat[kept], before[kept]), t
        assert torch.equal(pair.agents[1].partner_seat, pair.partner_seat)  # the BC agent plays agent 1's player


# ------------------------------------------------------------------------------------------------ whole windows


def _learner_rows(bp):
    T, n = bp.dones.shape
    return 2 * torch.arange(n, device="cuda") + (1 - bp.partner_seat.long())  # [T, N]


def _check_window(bs, bp, pair, lstm, with_seats):
    rows = _learner_rows(bp)
    for k in ("actions", "logp", "values", "rewards", "advantages", "value_targets"):
        assert torch.equal(getattr(bs, k).gather(1, rows), getattr(bp, k)), k
    assert torch.equal(bs.dones, bp.dones) and torch.equal(bs.states, bp.states)
    n = bp.dones.shape[1]
    after = 2 * torch.arange(n, device="cuda") + (1 - pair.partner_seat.long())
    assert torch.equal(bs.last_values[after], bp.last_values)
    if lstm:
        L = bp.seq_len
        for c in range(bp.state_h.shape[0]):
            assert torch.equal(bs.state_h[c][rows[c * L]], bp.state_h[c]) and torch.equal(bs.state_c[c][rows[c * L]], bp.state_c[c]), c
    fs, fp = bs.episodes.finished(), bp.episodes.finished()
    assert len(fp["ep_length"]) > 0
    for k in fs:
        if k != "partner_seat" or with_seats:
            assert torch.equal(fs[k], fp[k]), k
    if with_seats:
        assert torch.equal(bs.partner_seat, bp.partner_seat)


def _against_selfplay(make_env, A, seed, lstm, graph, T=30, windows=2, obs=False):
    e1, e2 = make_env(), make_env()
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=seed, use_graph=graph)
    pair = AgentPairRollout(e2, (A, copy.deepcopy(A)), seed=seed, use_graph=graph, random_seats=True)
    for w in range(windows):
        bs, bp = sp.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        assert bp.actions.shape == bp.dones.shape and torch.equal(bp.learner_mask, torch.ones_like(bp.dones))
        _check_window(bs, bp, pair, lstm, with_seats=False)
        assert torch.equal(e1.state, e2.state), w
        assert (bp.partner_seat == 0).any() and (bp.partner_seat == 1).any()
        if obs:
            n = e2.n_envs
            idx = torch.from_numpy(np.random.RandomState(w).choice(T * n, 200, replace=False)).cuda()
            p = (1 - bp.partner_seat.long()).view(-1)[idx]
            want = bs.observations(idx)[torch.arange(len(idx), device="cuda"), p]
            assert torch.equal(bp.observations(idx), want), w
    return pair


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pair_of_one_model_collects_what_selfplay_collects(lstm, graph):
    """(A, deepcopy(A)) with random seats: two windows whose episodes cross the window boundary equal self-play's windows
    at rows 2 e + p_t(e), including the bootstrap at the post-window seats and the LSTM state snapshots."""
    torch.manual_seed(3)
    A = RllibLSTMShapedCNN(5, 4) if lstm else RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", 517, horizon=20, auto_reset=True)
    pair = _against_selfplay(mk, A, 9, lstm, graph)
    assert all(a.fused_first_layer and a.fused_wide and a.fused_tail for a in pair.agents)


def test_library_path_learner_collects_what_selfplay_collects():
    """The nine 5x4 layouts with random_layout: more than K7 takes, so K2 -> the library layers on the learner's rows -> K8;
    batch.observations() is the learner's view of self-play's observations."""
    mk = lambda: BatchedOvercookedEnv(POOL_5X4, 300, horizon=7, auto_reset=True, random_layout=True, random_start_pos=True,
                                      rnd_obj_prob_thresh=0.6, seed=5)
    pair = _against_selfplay(mk, P.exact_cnn(5, 4, 21, cook_time=30), 4, False, True, T=12, obs=True)
    assert not pair.agents[0].fused_first_layer and pair.agents[0].fused_tail


def test_k7_only_learner_collects_what_selfplay_collects():
    """Dense layers of 128: K7 -> the library layers -> the one-view draw with logp."""
    mk = lambda: BatchedOvercookedEnv("cramped_room", 300, horizon=15, auto_reset=True)
    pair = _against_selfplay(mk, _exact_wide(5, 4, 3), 2, False, True, T=20, obs=True)
    assert pair.agents[0].fused_first_layer and not pair.agents[0].fused_tail


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pair_with_bc_collects_what_ppo_bc_collects(graph):
    """(A, bc) with random seats equals PPO_BC at bc_factor 1 on the learner's rows, the seats and the episode records over
    several episodes per environment."""
    n, horizon, T = 640, 12, 20
    torch.manual_seed(5)
    A, bc = RllibShapedCNN(5, 4), BCPolicy()
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=4, partner=copy.deepcopy(bc), bc_factor=1.0, use_graph=graph)
    pair = AgentPairRollout(e2, (A, bc), seed=4, random_seats=True, use_graph=graph)
    assert torch.equal(sp.partner_seat, pair.partner_seat)
    for w in range(2):
        bs, bp = sp.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        _check_window(bs, bp, pair, False, with_seats=True)
        assert torch.equal(e1.state, e2.state), w


def test_run_draws_what_collect_draws():
    n, T = 400, 25
    torch.manual_seed(6)
    A, B = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    p1 = AgentPairRollout(e1, (A, B), seed=8, random_seats=True)
    p2 = AgentPairRollout(e2, (copy.deepcopy(A), copy.deepcopy(B)), seed=8, random_seats=True)
    b = p1.collect(T, GAMMA, LAM)
    rows = _learner_rows(b)
    for t in range(T):
        assert torch.equal(p2.partner_seat, b.partner_seat[t].int()), t
        p2.run(1)
        assert torch.equal(p2.actions.view(-1)[rows[t]], b.actions[t]), t
    assert torch.equal(e1.state, e2.state) and torch.equal(p1.partner_seat, p2.partner_seat)


def test_reward_shaping_factor_reaches_the_captured_graph():
    n, T = 500, 30
    torch.manual_seed(7)
    A, B = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    pairs = [AgentPairRollout(BatchedOvercookedEnv("cramped_room", n, horizon=15, auto_reset=True), (copy.deepcopy(A), copy.deepcopy(B)),
                              seed=1, random_seats=True, use_graph=g) for g in (True, False)]
    for f in (1.0, 0.25):
        got = []
        for p in pairs:
            p.reward_shaping_factor = f
            b = p.collect(T, GAMMA, LAM)
            got.append((b.rewards.clone(), b.advantages.clone(), b.episodes.finished()["ep_reward_by_agent"]))
        for a, c in zip(*got):
            assert torch.equal(a, c), f
        assert pairs[0].reward_shaping_factor == f
    assert bool((got[0][0] % 1 != 0).any())  # shaped rewards of 3 / 5 at 0.25


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
def test_sync_weights_reaches_the_captured_window(lstm):
    """After sync_weights() the captured window equals a pair built fresh with the new learner weights from the same state;
    the partner draws what it drew before."""
    n, T = 300, 16
    torch.manual_seed(11)
    mk = (lambda: RllibLSTMShapedCNN(5, 4)) if lstm else (lambda: RllibShapedCNN(5, 4))
    A, B = mk(), mk()
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    pair = AgentPairRollout(e1, (A, B), seed=1, random_seats=True)
    pair.collect(T, GAMMA, LAM)  # captured with the old weights
    with torch.no_grad():
        for q in A.parameters():
            q.add_(torch.randn_like(q) * 0.05)
    pair.sync_weights()
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    fresh = AgentPairRollout(e2, (copy.deepcopy(A), copy.deepcopy(B)), seed=1, random_seats=True, use_graph=False)
    e2.state.copy_(e1.state), e2.done.copy_(e1.done)
    fresh.partner_seat.copy_(pair.partner_seat), fresh._seat_counter.copy_(pair._seat_counter)
    fresh.ret_sparse.copy_(pair.ret_sparse)
    for a, b in zip(fresh.stats.state_tensors(), pair.stats.state_tensors()):
        a.copy_(b)
    for fa, pa in zip(fresh.agents, pair.agents):
        fa._counter.copy_(pa._counter)
        fa.follow_seats()
        if lstm:
            fa.h.copy_(pa.h), fa.c.copy_(pa.c)
    bp = pair.collect(T, GAMMA, LAM)
    bf = fresh.collect(T, GAMMA, LAM)
    for k in ("actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "last_values", "partner_seat", "states"):
        assert torch.equal(getattr(bp, k), getattr(bf, k)), k
    assert torch.equal(e1.state, e2.state) and torch.equal(pair.actions, fresh.actions)
