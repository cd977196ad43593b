"""PPO sample batches on the device: the logp outputs of the draw kernels, ovc_record_transition, ovc_gae and
SelfPlayRollout.collect / sync_weights, against numpy restatements and the CPU oracle."""
import numpy as np
import pytest
import torch

from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout
from ppo_reference import gae_f32, gae_f64, log_softmax_at

pytestmark = pytest.mark.gpu


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _check_logp(logp, scores, actions, n_actions):
    want = log_softmax_at(scores, actions, n_actions)
    assert (np.abs(logp.astype(np.float64) - want) <= 1e-5 * (1 + np.abs(want))).all(), np.abs(logp - want).max()


@pytest.mark.parametrize("n_actions", [6, 7])
@pytest.mark.parametrize("n_rows", [1, 16, 4099])
def test_policy_tail_logp_is_policy_tail_plus_the_draws_log_probability(n_rows, n_actions):
    lib = _native.lib()
    rng = np.random.RandomState(n_rows + n_actions)
    k0, n_hidden = 160, 2
    x = _dev(rng.normal(size=(n_rows, k0)), torch.bfloat16)
    w1, b1 = _dev(rng.normal(size=(64, k0)) / np.sqrt(k0), torch.bfloat16), _dev(rng.normal(size=64) * 0.1, torch.float32)
    wh, bh = _dev(rng.normal(size=(n_hidden, 64, 64)) / 8, torch.bfloat16), _dev(rng.normal(size=(n_hidden, 64)) * 0.1, torch.float32)
    wo, bo = _dev(rng.normal(size=(8, 64)) / 2, torch.bfloat16), _dev(rng.normal(size=8) * 0.1, torch.float32)
    outs = []
    for with_logp in (False, True):
        counter = torch.zeros(2, dtype=torch.int64, device="cuda")
        actions = torch.full((n_rows,), -1, dtype=torch.int32, device="cuda")
        values = torch.zeros(n_rows, dtype=torch.float32, device="cuda")
        scores = torch.zeros((n_rows, 8), dtype=torch.float32, device="cuda")
        logp = torch.full((n_rows,), float("nan"), dtype=torch.float32, device="cuda")
        args = (x.data_ptr(), n_rows, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), n_hidden, wo.data_ptr(), bo.data_ptr(),
                0.3, n_actions, 1234, counter.data_ptr(), actions.data_ptr(), values.data_ptr(), scores.data_ptr())
        for _ in range(2):  # the second launch draws at step 1
            if with_logp:
                _native.check(lib.ovc_policy_tail_logp(*args, logp.data_ptr(), 0))
            else:
                _native.check(lib.ovc_policy_tail(*args, 0))
        assert _np(counter).tolist() == [2, 0]
        outs.append([_np(t) for t in (actions, values, scores, logp)])
    (a0, v0, s0, _), (a1, v1, s1, lp) = outs
    assert np.array_equal(a0, a1) and np.array_equal(v0, v1) and np.array_equal(s0, s1)
    assert a1.min() >= 0 and a1.max() < n_actions
    _check_logp(lp, s1, a1, n_actions)


@pytest.mark.parametrize("n_actions", [6, 8])
@pytest.mark.parametrize("n_rows", [1, 4099])
def test_sample_actions_logp_is_sample_actions_plus_the_draws_log_probability(n_rows, n_actions):
    lib = _native.lib()
    rng = np.random.RandomState(n_rows)
    scores = _dev(rng.normal(size=(n_rows, 8)) * 2, torch.float32)
    outs = []
    for with_logp in (False, True):
        counter = torch.zeros(2, dtype=torch.int64, device="cuda")
        actions = torch.full((n_rows,), -1, dtype=torch.int32, device="cuda")
        logp = torch.full((n_rows,), float("nan"), dtype=torch.float32, device="cuda")
        for _ in range(2):
            if with_logp:
                _native.check(lib.ovc_sample_actions_logp(scores.data_ptr(), 8, n_actions, n_rows, 77, counter.data_ptr(), actions.data_ptr(),
                                                          logp.data_ptr(), 0))
            else:
                _native.check(lib.ovc_sample_actions(scores.data_ptr(), 8, n_actions, n_rows, 77, counter.data_ptr(), actions.data_ptr(), 0))
        outs.append((_np(actions), _np(logp)))
    assert np.array_equal(outs[0][0], outs[1][0])
    _check_logp(outs[1][1], _np(scores), outs[1][0], n_actions)
    # the env wrapper: the same draw and logp for the 6 actions of the game
    env = BatchedOvercookedEnv("cramped_room", 8, horizon=400)
    sc = _dev(rng.normal(size=(16, 6)), torch.float32)
    lp = torch.empty(16, dtype=torch.float32, device="cuda")
    a = env.sample_actions(sc, torch.zeros(2, dtype=torch.int64, device="cuda"), seed=3, logp_out=lp)
    b = env.sample_actions(sc, torch.zeros(2, dtype=torch.int64, device="cuda"), seed=3)
    assert torch.equal(a, b)
    _check_logp(_np(lp), _np(sc), _np(a).reshape(-1), 6)


@pytest.mark.parametrize("gamma,lam", [(0.99, 0.95), (0.99, 1.0), (0.0, 0.95)])
@pytest.mark.parametrize("R", [2, 6002])
@pytest.mark.parametrize("T", [1, 7, 400])
def test_gae_kernel_bit_exact_vs_float32_loop(T, R, gamma, lam):
    rng = np.random.RandomState(T + R)
    rewards = rng.normal(size=(T, R)).astype(np.float32)
    values = rng.normal(size=(T, R)).astype(np.float32)
    last = rng.normal(size=R).astype(np.float32)
    dones = (rng.rand(T, R // 2) < 0.05).astype(np.uint8)
    dones[0, 0] = 1
    dones[T - 1, (R // 2) - 1] = 1
    env = BatchedOvercookedEnv("cramped_room", R // 2, horizon=400)
    adv, tgt = env.gae(_dev(rewards, torch.float32), _dev(values, torch.float32), _dev(dones, torch.uint8), _dev(last, torch.float32), gamma, lam)
    want_adv, want_tgt = gae_f32(rewards, values, dones, last, gamma, lam)
    assert np.array_equal(_np(adv), want_adv) and np.array_equal(_np(tgt), want_tgt)
    w64, t64 = gae_f64(rewards, values, dones, last, gamma, lam)
    assert (np.abs(_np(adv) - w64) <= 1e-5 * (1 + np.abs(w64))).all()


def test_record_transition_writes_rewards_and_dones_and_keeps_the_returns():
    n = 3001
    env = BatchedOvercookedEnv("cramped_room", n, horizon=30, auto_reset=True)
    twin = BatchedOvercookedEnv("cramped_room", n, horizon=30, auto_reset=True)
    rng = np.random.RandomState(4)
    factor = torch.full((1,), 0.75, dtype=torch.float32, device="cuda")
    rs, rm = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.float32, device="cuda")
    rs2, rm2 = rs.clone(), rm.clone()
    rewards, dones = torch.empty((n, 2), dtype=torch.float32, device="cuda"), torch.empty(n, dtype=torch.uint8, device="cuda")
    for t in range(70):
        a = rng.randint(0, 6, size=(n, 2)).astype(np.int32)
        sp, sh, dn, _ = [_np(x) for x in env.step(_dev(a, torch.int32))]
        twin.step(_dev(a, torch.int32))
        env.record_transition(factor, rewards=rewards, dones=dones, ret_sparse=rs, ret_mixed=rm)
        twin.accumulate_returns(rs2, rm2, 0.75)
        want = sp[:, None].astype(np.float32) + np.float32(0.75) * sh.astype(np.float32)
        assert np.array_equal(_np(rewards), want) and np.array_equal(_np(dones), (dn != 0).astype(np.uint8))
    assert torch.equal(rs, rs2) and torch.equal(rm, rm2)


def _oracle_check(env, s0, b, horizon, factor):
    """states[t] follow the oracle on actions[t] from s0, rewards / dones are the oracle's; returns the final state."""
    T, N = b.dones.shape
    ref = s0.copy()
    st, ac, rw, dn = _np(b.states), _np(b.actions), _np(b.rewards), _np(b.dones)
    assert (dn != 0).any(), "the window must cross episode ends"
    for t in range(T):
        assert np.array_equal(st[t], ref), t
        sp, sh, d, _ = cpu.step(env._tab_host, env._starts_host, ref, ac[t].reshape(N, 2), horizon=horizon, flags=1)
        want = sp[:, None].astype(np.float32) + np.float32(factor) * sh.astype(np.float32)
        assert np.array_equal(rw[t].reshape(N, 2), want) and np.array_equal(dn[t], (d != 0).astype(np.uint8)), t
    assert np.array_equal(_np(env.state), ref)
    return ref


def _fresh_eval(layout, n, horizon, model, state, step, seed):
    """actions, values, heads of a new SelfPlayRollout on ``state`` with its draw counter at ``step`` (one run())."""
    env = BatchedOvercookedEnv(layout, n, horizon=horizon, auto_reset=True)
    env.state.copy_(state)
    sp = SelfPlayRollout(env, model=model, use_graph=False, seed=seed)
    sp._draw_counter[0] = step
    if sp.fused_tail:
        sp._scores8 = torch.zeros((2 * n, 8), dtype=torch.float32, device="cuda")
    sp.run(1)
    heads = sp._scores8 if sp.fused_tail else sp._scores
    return _np(sp.actions).reshape(-1), _np(sp.values).reshape(-1), _np(heads)


@pytest.mark.parametrize("layout,flags", [("cramped_room", (True, True, True)), ("coordination_ring", (True, False, False)),
                                          ("asymmetric_advantages", (False, False, False))])
def test_collect_is_run_plus_the_sample_batch(layout, flags):
    n, T, H, seed, f = 300, 30, 13, 5, 0.5
    gamma, lam = 0.99, 0.95
    torch.manual_seed(3)
    W, Hh = {"cramped_room": (5, 4), "coordination_ring": (5, 5), "asymmetric_advantages": (9, 5)}[layout]
    model = RllibShapedCNN(W, Hh).cuda()
    envs = [BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True) for _ in range(3)]
    sps = [SelfPlayRollout(e, model=model, use_graph=g, seed=seed, reward_shaping_factor=f) for e, g in zip(envs, (True, False, True))]
    sp, sp_eager, sp_run = sps
    assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == flags
    for e in envs:
        e.rollout(torch.zeros((3, n, 2), dtype=torch.int32, device="cuda"))  # start all three mid-episode, alike
    s0 = _np(envs[0].state).copy()
    b = sp.collect(T, gamma, lam, keep_logits=True)
    assert np.array_equal(_np(b.states[0]), s0)
    _oracle_check(envs[0], s0, b, H, f)
    # run() from the same seed and counter: the same draws, the same end state, the same returns
    sp_run.run(T)
    assert torch.equal(envs[2].state, envs[0].state) and torch.equal(sp_run.actions.view(-1), b.actions[T - 1])
    assert torch.equal(sp_run._draw_counter, sp._draw_counter)
    assert torch.equal(sp_run.ret_sparse, sp.ret_sparse) and torch.equal(sp_run.ret_mixed, sp.ret_mixed)
    # eager == graph, every tensor of the batch
    be = sp_eager.collect(T, gamma, lam, keep_logits=True)
    for k in ("states", "actions", "logp", "values", "rewards", "dones", "last_values", "advantages", "value_targets", "logits"):
        assert torch.equal(getattr(be, k), getattr(b, k)), k
    assert torch.equal(envs[1].state, envs[0].state) and torch.equal(sp_eager.ret_mixed, sp.ret_mixed)
    # values / logp at slot t == a fresh evaluation of states[t] with the counter at t
    for t in (0, 7, T - 1):
        a, v, heads = _fresh_eval(layout, n, H, model, b.states[t], t, seed)
        assert np.array_equal(a, _np(b.actions[t])) and np.array_equal(v, _np(b.values[t])), t
        assert np.array_equal(heads[:, :6], _np(b.logits[t])[:, :6]), t
        _check_logp(_np(b.logp[t]), heads, a, 6)
    _, v, _ = _fresh_eval(layout, n, H, model, envs[0].state, 0, seed)
    assert np.array_equal(v, _np(b.last_values))
    adv, tgt = gae_f32(_np(b.rewards), _np(b.values), _np(b.dones), _np(b.last_values), gamma, lam)
    assert np.array_equal(_np(b.advantages), adv) and np.array_equal(_np(b.value_targets), tgt)
    # observations(): K2 of the stored records, both views, fp32 and bf16, == the oracle's encoding of the live state
    idx = torch.tensor([0, 5, 7 * n + 3, (T - 1) * n + n - 1], dtype=torch.int64, device="cuda")
    st = _np(b.states).reshape(T * n, -1)[_np(idx)]
    want = cpu.encode_lossless(envs[0]._tab_host, np.ascontiguousarray(st), W, Hh, horizon=H).astype(np.float32)
    for dt in (torch.float32, torch.bfloat16):
        obs = b.observations(idx, dtype=dt)
        assert obs.dtype == dt and tuple(obs.shape) == (4, 2, W, Hh, 26)
        assert np.array_equal(_np(obs.float()), want)
    live = BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True)
    live.state.copy_(b.states[7])
    assert torch.equal(b.observations(7 * n + torch.arange(n, device="cuda")), live.lossless_state_encoding())


def test_sync_weights_and_shaping_factor_reach_the_captured_graphs():
    layout, n, T, H, seed = "cramped_room", 300, 20, 11, 9
    torch.manual_seed(4)
    model = RllibShapedCNN(5, 4).cuda()
    env = BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True)
    sp = SelfPlayRollout(env, model=model, seed=seed, reward_shaping_factor=1.0)
    sp.run(2)  # run()'s graph, captured with the first weights
    run_graph = sp.graph
    sp.collect(T, 0.99, 0.95)
    graph = sp._collect_graphs[(T, False)][1]
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn_like(p) * 0.05)
    sp.sync_weights()
    s0, step = env.state.clone(), int(sp._draw_counter[0])
    b = sp.collect(T, 0.99, 0.95)
    a, v, _ = _fresh_eval(layout, n, H, model, s0, step, seed)
    assert np.array_equal(v, _np(b.values[0])) and np.array_equal(a, _np(b.actions[0]))
    s1, step = env.state.clone(), int(sp._draw_counter[0])
    sp.run(1)
    a, v, _ = _fresh_eval(layout, n, H, model, s1, step, seed)
    assert np.array_equal(v, _np(sp.values).reshape(-1)) and np.array_equal(a, _np(sp.actions).reshape(-1))
    # a new shaping factor reaches collect()'s graph and run()'s without a re-capture
    sp.reward_shaping_factor = 0.25
    s2 = _np(env.state).copy()
    b = sp.collect(T, 0.99, 0.95)
    assert sp._collect_graphs[(T, False)][1] is graph
    _oracle_check(env, s2, b, H, 0.25)
    shaped_seen = False
    for _ in range(200):  # until a step with shaped rewards has been checked
        before = _np(sp.ret_mixed).copy()
        sp.run(1)
        sh = _np(env.shaped).astype(np.float32)
        want = before + _np(env.sparse).astype(np.float32) + np.float32(0.25) * sh[:, 0] + np.float32(0.25) * sh[:, 1]
        assert np.array_equal(_np(sp.ret_mixed), want)
        shaped_seen = bool(sh.any())
        if shaped_seen:
            break
    assert sp.graph is run_graph and shaped_seen
