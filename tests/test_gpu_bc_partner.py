"""The behaviour-cloned partner of PPO_BC on the device: K10 (ovc_partner_policy) bit for bit against featurize_state of
the CPU oracle and a float64 restatement of the BC network on exactly representable operands (tests/policy_reference.py),
the seat draw (ovc_assign_partners) against a numpy Philox restatement, and SelfPlayRollout.run / collect with a partner."""
import numpy as np
import pytest
import torch

import policy_reference as P
import rollout_reference as R
from helpers import TRACE_FILES, TRACE_IDS, Trace
from oracle import cpu
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import PARTNER_DRAW_SALT, PARTNER_SEAT_SALT, BCPolicy, SelfPlayRollout
from ppo_reference import gae_f32
from rollout_reference import seats_reference

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 77


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _bc_operands(rng, n_hidden):
    """K10 tables as float64 arrays: K8's sparse dyadic tail operands over the 96 features."""
    _, w1, b1, wh, bh, wo, bo = P.k8_operands(rng, 0, 96, n_hidden)
    return w1, b1, wh, bh, wo, bo


def _tables(ops):
    return tuple(_dev(o, torch.bfloat16 if i % 2 == 0 else torch.float32) for i, o in enumerate(ops))


def _features(env, states):
    return R.features(env._tab_host, _np(env.feature_lut()), states)  # [N, 2, 96]


_heads = R.bc_heads


def _gumbel_rows(heads, rows, seed, step, n_actions):
    """gumbel_scores of the ovc_sample_actions definition on draw rows ``rows`` (not 0..len-1)."""
    big = np.zeros((int(rows.max()) + 1 if len(rows) else 1, 8))
    big[rows] = heads
    return P.gumbel_scores(big, seed, step, n_actions)[rows]


def _check_rows(actions, heads, rows, seed, step, n_actions):
    """actions == the draw on rows ``rows`` at ``step``, near-ties exempt."""
    if n_actions == 1 or len(rows) == 0:
        assert (actions == 0).all()
        return
    v = _gumbel_rows(heads, rows, seed, step, n_actions)
    top2 = np.sort(v, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-4  # libm and the device logf differ in the last bits: near-ties may flip
    assert clear.mean() > 0.99 and np.array_equal(actions[clear], v.argmax(1)[clear])
    assert actions.min() >= 0 and actions.max() < n_actions


def _k10_check(env, seats, ops, n_actions, seed=11, step=0):
    n = env.n_envs
    seat_t = _dev(seats, torch.int32)
    act_full = torch.full((n + GUARD, 2), SENTINEL, dtype=torch.int32, device="cuda")
    sc_full = torch.full((n + GUARD, 8), float("nan"), dtype=torch.float32, device="cuda")
    counter = torch.tensor([step, 0], dtype=torch.int64, device="cuda")
    env.partner_actions(_tables(ops), seat_t, counter, seed=seed, n_actions=n_actions, out=act_full[:n], scores=sc_full[:n])
    assert _np(counter).tolist() == [step + 1, 0]
    assert torch.equal(seat_t, _dev(seats, torch.int32))
    act, sc = _np(act_full), _np(sc_full)
    on = np.flatnonzero(seats >= 0)
    feats = _features(env, _np(env.state))[on, seats[on]]
    want = _heads(feats, ops)
    assert np.array_equal(sc[on], want), np.abs(sc[on] - want).max()
    _check_rows(act[on, seats[on]], want, 2 * on + seats[on], seed, step, n_actions)
    # untouched: self-play environments, the non-partner seat, everything past the end
    off = np.flatnonzero(seats < 0)
    assert (act[off] == SENTINEL).all() and np.isnan(sc[off]).all()
    assert (act[on, 1 - seats[on]] == SENTINEL).all()
    assert (act[n:] == SENTINEL).all() and np.isnan(sc[n:]).all()


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_k10_exact_on_fixture_states(path):
    tr = Trace(path)
    st = tr.data["obs_states"]
    env = BatchedOvercookedEnv(tr.layout, len(st), horizon=400)
    env.state.copy_(torch.from_numpy(st))
    rng = np.random.RandomState(len(st))
    seats = rng.randint(-1, 2, size=len(st)).astype(np.int32)
    _k10_check(env, seats, _bc_operands(rng, 1), 6)


POOL_5X4 = ["cramped_room", "cramped_room_tomato", "simple_o_t", "simple_tomato", "bonus_order_test", "mdp_test", "m_shaped_s",
            "simple_o", "cramped_room_o_3orders"]  # the 9 bundled two-player 5x4 layouts
K10_POOLS = {  # batches whose 64-environment tiles hold several layouts: (layouts, environment arguments for n envs)
    "interleaved": (["cramped_room", "mdp_test", "bonus_order_test", "m_shaped_s"], lambda n: {"env_layout": np.arange(n) % 4}),
    "pool_5x4_random_layout": (POOL_5X4, lambda n: {"random_layout": True, "horizon": 8}),  # 3 redraws in the 25 steps
    "mixed_shapes": (["cramped_room", "counter_circuit", "long_cook_time", "asymmetric_advantages_tomato"], lambda n: {}),
}


def _k10_pool_premises(env, seats):
    """Every layout occurs, some 64-environment tile holds more than one, and for some partnered environment layout 0's
    feature LUT gives other features than its own: a K10 that read the wrong layout's tables would fail."""
    st = _np(env.state)
    lid = st[:, 3] & 0xFF
    assert set(lid.tolist()) == set(range(env.n_layouts)), "premise: every layout occurs"
    assert any(len(np.unique(lid[i:i + 64])) > 1 for i in range(0, len(lid), 64)), "premise: a tile holds several layouts"
    lut = _np(env.feature_lut())
    on = np.flatnonzero(seats >= 0)
    right = cpu.featurize(env._tab_host, lut, st, num_pots=2)[on, seats[on]]
    wrong = cpu.featurize(env._tab_host, lut[np.zeros(env.n_layouts, np.int64)], st, num_pots=2)[on, seats[on]]
    assert (right != wrong).any(), "premise: layout 0's LUT featurizes no partnered environment differently"


@pytest.mark.parametrize("layout,n", [("long_cook_time", 777), ("counter_circuit", 1027), ("cramped_room", 2 * 333 + 1),
                                      ("interleaved", 779), ("pool_5x4_random_layout", 1001), ("mixed_shapes", 901)])
def test_k10_exact_on_random_rollouts(layout, n):
    """Random start states then random play; seats -1 / 0 / 1 mixed in each launch; n_hidden 0, 1, 2 and 1..7 actions;
    n is not a multiple of the 64-environment tile.  Several layouts per batch (``K10_POOLS``): env_layout interleaving
    four 5x4 layouts, the nine 5x4 layouts redrawn at every reset (random_layout), and four grid shapes in segments."""
    layouts, kw = K10_POOLS[layout] if layout in K10_POOLS else (layout, lambda n: {})
    kw = dict({"horizon": 60}, **kw(n))
    env = BatchedOvercookedEnv(layouts, n, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=n, **kw)
    rng = np.random.RandomState(n)
    acts = rng.randint(0, 6, size=(25, n, 2)).astype(np.int32)
    acts[rng.rand(25, n, 2) < 0.4] = 5
    env.rollout(torch.from_numpy(acts).cuda())
    for n_hidden in (0, 1, 2):
        for n_actions in range(1, 8):
            seats = rng.randint(-1, 2, size=n).astype(np.int32)
            _k10_check(env, seats, _bc_operands(rng, n_hidden), n_actions, seed=n_actions, step=n_hidden * 7 + n_actions)
    _k10_check(env, np.full(n, -1, np.int32), _bc_operands(rng, 1), 6)
    _k10_check(env, np.ones(n, np.int32), _bc_operands(rng, 1), 6)
    if layout in K10_POOLS:
        _k10_pool_premises(env, np.ones(n, np.int32))


def test_k10_exact_on_l16_features_above_256():
    """K10 on a 16x16 layout with 4 pots, of which featurize_state (num_pots = 2) shows the 2 nearest, and cook times up to
    16382: features above 256 that bfloat16 cannot hold reach the first layer rounded to nearest even."""
    import limit_layouts as LL
    from overcooked_ai_b200 import layout as L

    lay = LL.l16()
    n = 601
    env = BatchedOvercookedEnv(lay, n, horizon=60, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.8, seed=5)
    rng = np.random.RandomState(1)
    acts = rng.randint(0, 6, size=(40, n, 2)).astype(np.int32)
    acts[rng.rand(40, n, 2) < 0.4] = 5
    env.rollout(torch.from_numpy(acts).cuda())
    st = _np(env.state).copy()
    hand = np.stack([L.pack_state(lay, s, 0, env.state_words) for s in LL.l16_states(lay).values()])
    st[::40][:len(hand)] = hand
    env.state.copy_(torch.from_numpy(st))
    feats = _features(env, st).reshape(-1, 96)
    big = np.flatnonzero(np.abs(feats).max(0) > 256)  # the pots' cook time remaining, in both blocks
    assert len(big) and (P.bf16(feats) != feats).any(), "premise: some features are not exact in bfloat16"
    for n_hidden in (0, 1, 2):
        ops = list(_bc_operands(rng, n_hidden))
        ops[0] = ops[0].copy()
        ops[0][:, big] *= 2.0 ** -6  # keeps every accumulation exact with inputs up to 16384
        assert (ops[0][:, big] != 0).any()
        w1 = ops[0]
        assert not np.array_equal(feats @ w1.T, P.bf16(feats) @ w1.T), "premise: the rounding reaches the first layer"
        seats = rng.randint(-1, 2, size=n).astype(np.int32)
        seats[::40] = rng.randint(0, 2, size=len(seats[::40]))
        _k10_check(env, seats, tuple(ops), 6, seed=3, step=n_hidden)


def test_k10_draw_step_past_2_to_the_32():
    env = BatchedOvercookedEnv("cramped_room", 300, horizon=400, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=2)
    rng = np.random.RandomState(5)
    ops = _bc_operands(rng, 1)
    for step in (2**32 - 1, 2**32, 2**33 + 5):
        _k10_check(env, rng.randint(-1, 2, size=300).astype(np.int32), ops, 6, seed=99, step=step)


def test_k10_refuses_what_it_is_not_built_for():
    env = BatchedOvercookedEnv("cramped_room", 10, horizon=400)
    rng = np.random.RandomState(0)
    seat = torch.zeros(10, dtype=torch.int32, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    w1, b1, wh, bh, wo, bo = _tables(_bc_operands(rng, 1))
    with pytest.raises(RuntimeError, match="96 features"):
        env.partner_actions((w1[:, :64].contiguous(), b1, wh, bh, wo, bo), seat, counter)
    with pytest.raises(RuntimeError, match="n_actions"):
        env.partner_actions((w1, b1, wh, bh, wo, bo), seat, counter, n_actions=8)


# --------------------------------------------------------------------------------------------------- the seat draw
@pytest.mark.parametrize("n", [1, 255, 4099])
def test_assign_partners_matches_the_restatement(n):
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    rng = np.random.RandomState(n)
    full = torch.full((n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    seat = full[:n]
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    factor = torch.zeros(1, dtype=torch.float32, device="cuda")
    ref = np.full(n, SENTINEL, np.int32)
    for step, f, with_done in ((0, 0.0, False), (1, 1.0, False), (2, 0.3, True), (3, 0.7, True), (4, 1.0, True), (5, 0.0, True), (6, 0.55, False)):
        factor.fill_(f)
        done = (rng.rand(n) < 0.3).astype(np.int32) if with_done else None
        env.assign_partners(seat, factor, counter, seed=1234, done=None if done is None else _dev(done, torch.int32))
        ref = seats_reference(n, 1234, step, f, ref, done)
        got = _np(seat)
        assert np.array_equal(got, ref), step
        if f == 0.0:
            assert (got[done != 0] == -1).all() if done is not None else (got == -1).all()
        if f == 1.0:
            assert (got[done != 0] >= 0).all() if done is not None else (got >= 0).all()
        assert (_np(full[n:]) == SENTINEL).all()
    assert _np(counter).tolist() == [7, 0]
    if n == 4099:  # both seats and self-play occur at a fractional factor
        assert set(np.unique(ref).tolist()) == {-1, 0, 1}


def test_assign_partners_follows_a_factor_changed_between_graph_replays():
    n = 2000
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    seat = torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    factor = torch.zeros(1, dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        env.assign_partners(seat, factor, counter, seed=7)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.assign_partners(seat, factor, counter, seed=7)
    counter.zero_()
    for step, f in enumerate((0.0, 1.0, 0.25)):
        factor.fill_(f)
        g.replay()
        assert np.array_equal(_np(seat), seats_reference(n, 7, step, f, None)), f


# --------------------------------------------------------------------------------------------------- the rollout
def _exact_bc(rng):
    """A BCPolicy whose tables are the dyadic K10 operands (exact in bf16)."""
    w1, b1, wh, bh, wo, bo = _bc_operands(rng, 1)
    bc = BCPolicy()
    bc.load_keras_weights([(w1.T, b1), (wh[0].T, bh[0])], (wo[:6].T, bo[:6]))
    return bc, (w1, b1, wh, bh, np.concatenate([wo[:6], np.zeros((2, 64))]), np.concatenate([bo[:6], np.zeros(2)]))


def _ppo_draws(layout, n, horizon, model, state, step, seed):
    """The PPO policy's joint action on ``state`` with its draw counter at ``step``, without a partner."""
    env = BatchedOvercookedEnv(layout, n, horizon=horizon, auto_reset=True)
    env.state.copy_(state)
    sp = SelfPlayRollout(env, model=model, use_graph=False, seed=seed)
    sp._draw_counter[0] = step
    sp.run(1)
    return _np(sp.actions).reshape(-1)


@pytest.mark.parametrize("use_graph", [False, True])
def test_collect_with_a_bc_partner(use_graph):
    layout, n, T, H, seed = "cramped_room", 130, 30, 13, 21
    gamma, lam = 0.99, 0.95
    rng = np.random.RandomState(3)
    model = P.exact_cnn(5, 4, 8).cuda()
    bc, ops = _exact_bc(rng)
    envs = [BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True) for _ in range(2)]
    for e in envs:
        e.rollout(torch.zeros((4, n, 2), dtype=torch.int32, device="cuda"))
    sp = SelfPlayRollout(envs[0], model=model, use_graph=use_graph, seed=seed, partner=bc, bc_factor=0.6)
    sp_run = SelfPlayRollout(envs[1], model=model, use_graph=use_graph, seed=seed, partner=bc, bc_factor=0.6)
    s0 = _np(envs[0].state).copy()
    b = sp.collect(T, gamma, lam)
    st, ac, seat, dn = _np(b.states), _np(b.actions), _np(b.partner_seat).astype(np.int32), _np(b.dones)
    assert np.array_equal(st[0], s0) and (dn != 0).any()
    # the seats: every environment drawn at construction (step 0), then redrawn exactly where an episode ended
    assert np.array_equal(seat[0], seats_reference(n, seed ^ PARTNER_SEAT_SALT, 0, 0.6, None))
    for t in range(1, T):
        assert np.array_equal(seat[t], seats_reference(n, seed ^ PARTNER_SEAT_SALT, t, 0.6, seat[t - 1], dn[t - 1])), t
    assert (seat >= 0).any() and (seat < 0).any()
    mask = _np(b.learner_mask).reshape(T, n, 2)
    assert np.array_equal(mask, (seat[:, :, None] != np.arange(2)).astype(np.uint8))
    for t in range(T):
        # learner rows: what the PPO policy draws on states[t] without a partner
        ppo = _ppo_draws(layout, n, H, model, b.states[t], t, seed).reshape(n, 2)
        assert np.array_equal(ac[t].reshape(n, 2)[mask[t] == 1], ppo[mask[t] == 1]), t
        # partner rows: the BC restatement on featurize(states[t]), drawn at step t with the partner's key
        on = np.flatnonzero(seat[t] >= 0)
        feats = _features(envs[0], st[t])[on, seat[t][on]]
        _check_rows(ac[t].reshape(n, 2)[on, seat[t][on]], _heads(feats, ops), 2 * on + seat[t][on], seed ^ PARTNER_DRAW_SALT, t, 6)
    # advantages of learner rows: GAE run per episode on those rows alone
    rw, vl, adv, last = _np(b.rewards), _np(b.values), _np(b.advantages), _np(b.last_values)
    for e in range(n):
        ends = list(np.flatnonzero(dn[:, e])) + ([T - 1] if not dn[T - 1, e] else [])
        t0 = 0
        for t1 in ends:
            cols = [2 * e, 2 * e + 1]
            a, _ = gae_f32(rw[t0:t1 + 1, cols], vl[t0:t1 + 1, cols], dn[t0:t1 + 1, e:e + 1], last[cols], gamma, lam)
            keep = mask[t0:t1 + 1, e] == 1
            assert np.array_equal(adv[t0:t1 + 1, cols][keep], a[keep]), (e, t0, t1)
            t0 = t1 + 1
    # run() from the same seed and counters: the same draws, seats and end state
    sp_run.run(T)
    assert torch.equal(envs[1].state, envs[0].state) and torch.equal(sp_run.partner_seat, sp.partner_seat)
    assert np.array_equal(_np(sp_run.actions).reshape(-1), ac[T - 1])
    for k in ("_draw_counter", "_partner_counter", "_seat_counter"):
        assert torch.equal(getattr(sp_run, k), getattr(sp, k)), k
    # an annealed factor reaches the captured graphs: at 1, every episode that starts is partnered
    sp.bc_factor = 1.0
    b = sp.collect(T, gamma, lam)
    seat, dn = _np(b.partner_seat), _np(b.dones)
    started = np.cumsum(dn, 0)[:-1] > 0  # an episode ended before t
    assert (seat[1:][started] >= 0).all()


@pytest.mark.parametrize("use_graph", [False, True])
def test_a_partner_that_never_plays_changes_nothing(use_graph):
    """bc_factor = 0: K10 writes nothing and the rollout is the self-play rollout, draw for draw."""
    layout, n, T, H, seed = "cramped_room", 200, 25, 11, 4
    torch.manual_seed(1)
    from overcooked_ai_b200.selfplay import RllibShapedCNN
    model = RllibShapedCNN(5, 4).cuda()
    envs = [BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True) for _ in range(2)]
    sps = [SelfPlayRollout(envs[0], model=model, use_graph=use_graph, seed=seed),
           SelfPlayRollout(envs[1], model=model, use_graph=use_graph, seed=seed, partner=BCPolicy(), bc_factor=0.0)]
    b0, b1 = (sp.collect(T, 0.99, 0.95) for sp in sps)
    for k in ("states", "actions", "logp", "values", "rewards", "dones", "last_values", "advantages", "value_targets"):
        assert torch.equal(getattr(b0, k), getattr(b1, k)), k
    assert (b1.partner_seat == -1).all() and b1.learner_mask.all() and b0.partner_seat is None
    for sp in sps:
        sp.run(7)
    assert torch.equal(envs[0].state, envs[1].state) and torch.equal(sps[0].actions, sps[1].actions)
