"""SelfPlayRollout on layout pools (variable-MDP training: ``random_layout=True`` redraws an environment's layout at every
reset) and on batches that interleave layouts.  Every kernel of the PPO path reads the layout id from word 3 of each record:
K7 or K2, K1's redraw, K10 and the episode statistics.  collect()'s heads are compared with the float64 CNN on the
oracle's encoding of the batch's states, the window with the oracle's replay under the same random starts and redraws,
and the episode records, the seats and the BC partner's actions with their restatements.

Pools of 5x4 layouts: P9, the nine bundled ones (more than K7 takes per call: K2 -> library GEMMs -> K8); P8, eight of them
(K7 -> K9 -> K8); G12, twelve generated ones; and three layouts interleaved by env_layout, without redraws."""
import math

import numpy as np
import pytest
import torch

import policy_reference as P
from episode_reference import EpisodeReference, rewards_f32
from oracle import cpu
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.layout_generator import generate_layout_pool
from overcooked_ai_b200.selfplay import PARTNER_DRAW_SALT, PARTNER_SEAT_SALT, SelfPlayRollout
from test_gpu_bc_partner import POOL_5X4, _check_rows, _exact_bc, _features, _heads, _ppo_draws, seats_reference
from test_gpu_episode_stats import _check_equal, _records_equal

pytestmark = pytest.mark.gpu

HORIZON = 7
THRESH = 0.6
COOK = 30  # the longest cook time of the bundled 5x4 layouts (cramped_room_tomato): bounds the exact CNN's inputs
INTERLEAVED = ["cramped_room", "mdp_test", "bonus_order_test"]
FUSED, LIBRARY = (True, True, True), (False, False, True)  # (fused_first_layer, fused_wide, fused_tail)


def _np(t):
    return t.cpu().numpy()


def _g12():
    saved = np.random.get_state()
    np.random.seed(7)  # generate_layout_pool draws from numpy's global generator
    try:
        return generate_layout_pool(12, outer_shape=(5, 4))
    finally:
        np.random.set_state(saved)


POOLS = {"P9": lambda: POOL_5X4, "P8": lambda: POOL_5X4[:8], "G12": _g12, "interleaved": lambda: INTERLEAVED}


def _env(pool, n, seed):
    """Random starts with objects (so that short episodes deliver), horizon 7: a window of a dozen transitions crosses
    every environment's episode end at least once."""
    layouts = POOLS[pool]()
    inter = pool == "interleaved"
    return BatchedOvercookedEnv(layouts, n, horizon=HORIZON, auto_reset=True, random_layout=not inter,
                                env_layout=np.arange(n) % len(layouts) if inter else None, random_start_pos=True,
                                rnd_obj_prob_thresh=THRESH, seed=seed)


def _load(dst, src):
    with torch.no_grad():
        for p, q in zip(dst.parameters(), src.parameters()):
            p.copy_(q)


def _replay(env, b, seed, ref=None):
    """states[t] follow the oracle from states[0] on actions[t], with the device's random starts and layout redraws
    (``seed`` = the environment's); rewards and dones are the oracle's.  Feeds ``ref`` (an EpisodeReference) when given.
    Returns the number of deliveries on an episode's last transition whose value on the layout the episode was played on
    differs from the value on the layout the environment is redrawn to."""
    T, N = b.dones.shape
    rs = cpu.random_start(seed, THRESH, True, env.random_layout)
    st, ac, rw, dn = _np(b.states), _np(b.actions), _np(b.rewards), _np(b.dones)
    seat = None if b.partner_seat is None else _np(b.partner_seat).astype(np.int32)
    vals = np.stack([l.deliver_value for l in env.layouts])
    state = st[0].copy()
    if ref is not None:
        ref.clear()
    misattributable = 0
    for t in range(T):
        assert np.array_equal(st[t], state), t
        before = state[:, 3] & 0xFF
        sp, sh, d, ev = cpu.step(env._tab_host, env._starts_host, state, ac[t].reshape(N, 2), horizon=HORIZON, flags=1, rs=rs)
        after = state[:, 3] & 0xFF
        assert np.array_equal(rw[t].reshape(N, 2), rewards_f32(sp, sh, 1.0)), t
        assert np.array_equal(dn[t], (d != 0).astype(np.uint8)), t
        if ref is not None:
            ref.step(sh, d, ev, after, rw[t].reshape(N, 2), None if seat is None else seat[t])
        rec = (ev >> 25) & 15
        last = ((ev >> 15) & 1).astype(bool) & (d != 0)[:, None]
        misattributable += int((last & (vals[before[:, None], rec] != vals[after[:, None], rec])).sum())
    assert np.array_equal(_np(env.state), state)
    return misattributable


def _check_heads(b, env, cnn, seed, step0):
    """logits / values / last_values == the float64 CNN on the oracle's encoding of states[t] (and of the state after the
    window), logp to 1e-5, actions the draw at step step0 + t; observations() is the oracle's encoding."""
    T, N = b.dones.shape
    obs = cpu.encode_lossless(env._tab_host, _np(b.states).reshape(T * N, -1), 5, 4, horizon=HORIZON)
    assert obs.min() >= 0 and (obs <= P.plane_bounds(COOK)).all(), "premise: an observation exceeds the planes' bounds"
    assert np.array_equal(_np(b.observations(torch.arange(T * N, device="cuda"))), obs.astype(np.float32))
    logits, values = P.cnn_forward64(cnn, obs)
    logits, values = logits.reshape(T, 2 * N, 6), values.reshape(T, 2 * N)
    assert np.array_equal(_np(b.logits)[..., :6], logits) and np.array_equal(_np(b.values), values)
    for t in range(T):
        P.check_draw(_np(b.actions[t]), logits[t], seed, step0 + t)
        P.check_logp(_np(b.logp[t]), logits[t], _np(b.actions[t]), 6)
    last = cpu.encode_lossless(env._tab_host, _np(env.state), 5, 4, horizon=HORIZON)
    assert np.array_equal(_np(b.last_values), P.cnn_forward64(cnn, last)[1])
    assert len(np.unique(logits)) > 8 and len(np.unique(_np(b.actions))) == 6


def _check_layouts(env, b):
    """Every layout of the pool occurs in the window; with random_layout the ids change within it, interleaved they stay."""
    lid = _np(b.states)[..., 3] & 0xFF
    assert set(np.unique(lid).tolist()) == set(range(env.n_layouts))
    if env.random_layout:
        assert (lid != lid[:1]).any()
    else:
        assert (lid == env.env_layout_host).all()


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("pool,flags", [("P8", FUSED), ("P9", LIBRARY), ("G12", LIBRARY), ("interleaved", FUSED)])
def test_collect_on_a_pool_is_the_float64_cnn_and_the_oracle(pool, flags, use_graph):
    """collect() on a pool, exact weights: the heads equal the float64 CNN on the oracle's encoding of the batch's states and
    the window equals the oracle's replay with the same random starts and redraws; after a second network is loaded and
    sync_weights() called, the next window (the same captured graph) equals the new network."""
    n, T, seed, env_seed = 777, 16, 4, 11
    model = P.exact_cnn(5, 4, 21, cook_time=COOK).cuda()
    env = _env(pool, n, env_seed)
    sp = SelfPlayRollout(env, model=model, use_graph=use_graph, seed=seed)
    second = P.exact_cnn(5, 4, 22, cook_time=COOK)
    for w, cnn in enumerate((model, second)):
        if w:
            graph = sp._collect_graphs.get((T, True))
            _load(model, second)
            sp.sync_weights()
        step0 = int(sp._draw_counter[0])
        b = sp.collect(T, 0.99, 0.95, keep_logits=True)
        assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == flags
        if w:
            assert sp._collect_graphs.get((T, True)) is graph
        _check_layouts(env, b)
        _replay(env, b, env_seed)
        _check_heads(b, env, cnn, seed, step0)


def test_k7_is_refused_on_more_than_8_layouts_when_the_rollout_is_built():
    env = _env("P9", 65, 1)
    with pytest.raises(AssertionError, match="at most 8 layouts"):
        SelfPlayRollout(env, fused_first_layer=True)
    with pytest.raises(AssertionError, match="K9 sits between K7 and K8"):
        SelfPlayRollout(env, fused_wide=True)
    sp = SelfPlayRollout(env, use_graph=False)
    assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == LIBRARY
    sp.run(2)  # the default path runs


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("pool", ["P9", "P8"])
def test_episodes_and_bc_partner_on_a_pool(pool, use_graph):
    """A BC partner at bc_factor 0.6 on a pool with random_layout, three windows of 12 transitions (episodes of 7 cross
    the window boundaries): b.episodes and the running statistics equal EpisodeReference fed by the oracle's replay with
    the pool's own delivery values, the seats equal the seat draw's restatement, partner rows the BC restatement on
    featurize(states[t]), learner rows the PPO draws without a partner; run() from the same seed leaves the same state,
    seats, counters and records.  Premises: episodes start on another layout than their environment's at the window's
    start, and deliveries on an episode's last transition are worth something else on the layout the environment moves to."""
    n, T, seed, env_seed, factor = 2048, 12, 13, 9, 0.6
    cap = math.ceil(T / HORIZON)
    rng = np.random.RandomState(3)
    model = P.exact_cnn(5, 4, 8, cook_time=COOK).cuda()
    bc, ops = _exact_bc(rng)
    envs = [_env(pool, n, env_seed) for _ in range(2)]
    sp = SelfPlayRollout(envs[0], model=model, use_graph=use_graph, seed=seed, partner=bc, bc_factor=factor)
    sp_run = SelfPlayRollout(envs[1], model=model, use_graph=use_graph, seed=seed, partner=bc, bc_factor=factor, episode_capacity=cap)
    vals = np.stack([l.deliver_value for l in envs[0].layouts])
    assert len({tuple(v) for v in vals}) > 4
    ref = EpisodeReference(vals, _np(envs[0].state)[:, 3] & 0xFF, cap)
    prev_seat = prev_done = None
    moved = misattributable = 0
    for w in range(3):
        b = sp.collect(T, 0.99, 0.95)
        st, ac, seat, dn = _np(b.states), _np(b.actions), _np(b.partner_seat).astype(np.int32), _np(b.dones)
        _check_layouts(envs[0], b)
        lid = st[..., 3] & 0xFF
        moved += int(((dn[:-1] != 0) & (lid[1:] != lid[:1])).sum())  # an episode starts at t on another layout than at 0
        misattributable += _replay(envs[0], b, env_seed, ref)
        _check_equal(sp.stats, b.episodes, ref)
        assert not ref.dropped.any() and ref.count.sum() > 0
        for t in range(T):
            step = w * T + t
            want = seats_reference(n, seed ^ PARTNER_SEAT_SALT, step, factor, prev_seat, prev_done)
            assert np.array_equal(seat[t], want), (w, t)
            prev_seat, prev_done = seat[t], dn[t]
            on = np.flatnonzero(seat[t] >= 0)
            feats = _features(envs[0], st[t])[on, seat[t][on]]
            _check_rows(ac[t].reshape(n, 2)[on, seat[t][on]], _heads(feats, ops), 2 * on + seat[t][on], seed ^ PARTNER_DRAW_SALT, step, 6)
            mask = seat[t][:, None] != np.arange(2)
            ppo = _ppo_draws(envs[0].layouts, n, HORIZON, model, b.states[t], step, seed).reshape(n, 2)
            assert np.array_equal(ac[t].reshape(n, 2)[mask], ppo[mask]), (w, t)
        assert (seat >= 0).any() and (seat < 0).any()
        sp_run.episodes.clear()
        sp_run.run(T)
        assert torch.equal(envs[1].state, envs[0].state) and torch.equal(sp_run.partner_seat, sp.partner_seat)
        for k in ("_draw_counter", "_partner_counter", "_seat_counter"):
            assert torch.equal(getattr(sp_run, k), getattr(sp, k)), k
        _records_equal(sp_run.episodes, b.episodes)
        for x, y in zip(sp_run.stats.state_tensors(), sp.stats.state_tensors()):
            assert torch.equal(x, y)
    assert moved > 0, "premise: no episode started on another layout"
    assert misattributable > 0, "premise: no delivery whose value depends on the layout it is credited to"
