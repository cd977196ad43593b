"""The potential-based dense reward (use_phi) on the device: ovc_potential_shaping against the CPU oracle,
ovc_record_transition_dense against a numpy restatement, and SelfPlayRollout / AgentPairRollout with use_phi against the
same rollouts without it, an oracle replay and BatchedOvercookedMultiAgent(use_phi=True).  Bit for bit throughout."""
import copy

import numpy as np
import pytest
import torch

import limit_layouts as LL
from helpers import GOLD, Trace
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeRecords, EpisodeStats
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout
from overcooked_ai_b200.vecenv import BatchedOvercookedMultiAgent
from ppo_reference import gae_f32
from test_gpu_pair_collect import _check_window

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _phi(env, recs):
    pt, cl, gpow = L.build_potential_tables(env.layouts, 0.99)
    return cpu.potential(env._tab_host, pt, cl, gpow, recs)


# ------------------------------------------------------------------------------------------------ ovc_potential_shaping


def _pool():
    from overcooked_ai_b200 import layout_generator as LG

    np.random.seed(5)
    params = {"inner_shape": (6, 5), "prop_empty": 0.6, "prop_feats": 0.3, "display": False, "feature_types": ["P", "D", "S", "O", "T"],
              "start_all_orders": [{"ingredients": ["onion", "tomato"]}, {"ingredients": ["onion", "onion", "onion"]}]}
    return LG.generate_layout_pool(5, params, outer_shape=(7, 6), skip_unsupported=True)


CASES = {
    "standard": lambda: (["cramped_room"], {}),
    "random_start": lambda: (["cramped_room"], dict(random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=7)),
    "layout_pool": lambda: (_pool(), dict(random_layout=True, random_start_pos=True, seed=5)),
    "limits": lambda: ([LL.l16(), LL.l3p()], {}),
}


def _start_states(case, env, rng, H):
    """Records to start from: the cramped_room trace fixture's states, or the env's own after random play; timesteps
    drawn below the horizon so that episodes end throughout the test."""
    n = env.n_envs
    if case == "standard":
        st = Trace(GOLD + "/trace_cramped_room.npz").data["obs_states"]
        st = np.ascontiguousarray(np.resize(st, (n, st.shape[1])))
    else:
        env.rollout(_dev(rng.randint(0, 6, size=(5, n, 2)), torch.int32))
        st = _np(env.state).copy()
        if case == "limits":
            lay = env.layouts[0]
            special = [L.pack_state(lay, s, 0, env.state_words) for s in LL.l16_states(lay).values()]
            st[:len(special)] = np.stack(special)
    st[:, 0] = rng.randint(0, H, size=n)
    return st


def _shaping(env, phi_s, dense, n):
    """ovc_potential_shaping on the first n environments only (the rest are sentinels)."""
    pt, cl, gpow = env.potential_tables(0.99)
    _native.check(env._lib.ovc_potential_shaping(
        env.tables.data_ptr(), env.n_layouts, env.start_records.data_ptr(), pt.data_ptr(), cl.data_ptr(), gpow.data_ptr(), gpow.numel(),
        env.state.data_ptr(), env.done.data_ptr(), phi_s.data_ptr(), dense.data_ptr(), n, env.state_words, env._rs_ptr(), env._stream()))


@pytest.mark.parametrize("case", list(CASES))
def test_potential_shaping_vs_oracle(case):
    """dense = float32(phi(s') - phi(s)) on the record the step left, then the reset an auto_reset env makes; the
    environments past n keep their terminal record and their dense sentinel."""
    layouts, kw = CASES[case]()
    n, pad, H, T = 1021, 8, 6, 20
    rng = np.random.RandomState(len(case))
    env = BatchedOvercookedEnv(layouts, n + pad, horizon=H, auto_reset=True, **kw)
    twin = BatchedOvercookedEnv(layouts, n + pad, horizon=H, auto_reset=True, **kw)
    s0 = _start_states(case, env, rng, H)
    env.state.copy_(torch.from_numpy(s0)), twin.state.copy_(torch.from_numpy(s0))
    phi_s = torch.empty(n + pad, dtype=torch.float64, device="cuda")
    ended = 0
    for t in range(T):
        a = rng.randint(0, 6, size=(n + pad, 2)).astype(np.int32)
        s = _np(env.state).copy()
        env.potential(0.99, out=phi_s)
        env.step(_dev(a, torch.int32), auto_reset=False)
        term = _np(env.state).copy()
        ref = s.copy()
        _, _, done, _ = cpu.step(env._tab_host, env._starts_host, ref, a, horizon=H, flags=0)
        assert np.array_equal(term, ref) and np.array_equal(_np(env.done), done), t
        dense = torch.full((n + pad,), 7.5, dtype=torch.float32, device="cuda")
        _shaping(env, phi_s, dense, n)
        want = (_phi(env, term) - _phi(env, s)).astype(np.float32)
        got = _np(dense)
        assert np.array_equal(got[:n], want[:n]) and (got[n:] == 7.5).all(), t
        twin.step(_dev(a, torch.int32))
        st = _np(env.state)
        assert np.array_equal(st[:n], _np(twin.state)[:n]) and np.array_equal(st[n:], term[n:]), t
        env.state[n:] = twin.state[n:]
        ended += int(done[:n].sum())
    assert ended > n and (want != 0).any()


# ------------------------------------------------------------------------------------------------ ovc_record_transition_dense


@pytest.mark.parametrize("stats", [False, True], ids=["plain", "stats"])
@pytest.mark.parametrize("one_view", [False, True], ids=["two_rows", "one_view"])
def test_record_transition_dense_vs_restatement(one_view, stats):
    """rewards, ret_mixed and reward_by_agent follow the dense reward; dones, ret_sparse and every other statistic and
    record are what ovc_record_transition_stats writes from the same step."""
    n, H, f, cap = 3001, 9, 0.75, 5
    env = BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True)
    rng = np.random.RandomState(11)
    factor = torch.full((1,), f, dtype=torch.float32, device="cuda")
    rewards = torch.empty((n,) if one_view else (n, 2), dtype=torch.float32, device="cuda")
    side = [dict(dones=torch.empty(n, dtype=torch.uint8, device="cuda"), ret_sparse=torch.zeros(n, dtype=torch.int64, device="cuda"),
                 ret_mixed=torch.zeros(n, dtype=torch.float32, device="cuda")) for _ in range(2)]
    if stats:
        ps = _dev(rng.randint(-1, 2, size=n), torch.int32)
        for kw in side:
            kw.update(stats=EpisodeStats(env), records=EpisodeRecords(env, cap), partner_seat=ps)
    want_rm, run_rw = np.zeros(n, np.float32), np.zeros(n, np.float32)
    want_rec, cnt = np.zeros((cap, n), np.float32), np.zeros(n, np.int64)
    for t in range(4 * H):
        env.step(_dev(rng.randint(0, 6, size=(n, 2)), torch.int32))
        d = (rng.normal(size=n) * 3).astype(np.float32)
        if one_view:
            env.record_transition_view(factor, 0, None, rewards, dense=_dev(d, torch.float32), **side[0])
        else:
            env.record_transition(factor, rewards=rewards, dense=_dev(d, torch.float32), **side[0])
        env.record_transition(factor, **side[1])
        sp, done = _np(env.sparse).astype(np.float32), _np(env.done) != 0
        fd = np.float32(f) * d
        r = sp + fd
        want_rm = ((want_rm + sp) + fd) + fd
        assert np.array_equal(_np(rewards), r if one_view else np.stack([r, r], 1)), t
        assert np.array_equal(_np(side[0]["ret_mixed"]), want_rm), t
        for k in ("dones", "ret_sparse"):
            assert torch.equal(side[0][k], side[1][k]), (k, t)
        run_rw = run_rw + r
        for e in np.nonzero(done)[0]:
            if cnt[e] < cap:
                want_rec[cnt[e], e] = run_rw[e]
            cnt[e] += 1
        run_rw[done] = 0
    if not stats:
        return
    a, b = side
    assert np.array_equal(_np(a["stats"].ep_reward_by_agent), np.stack([run_rw, run_rw], 1))
    for x, y in zip(a["stats"].state_tensors(), b["stats"].state_tensors()):
        if x is not a["stats"].ep_reward_by_agent:
            assert torch.equal(x, y)
    for x, y in zip(a["records"].tensors(), b["records"].tensors()):
        if x is not a["records"].reward_by_agent:
            assert torch.equal(x, y)
    assert np.array_equal(_np(a["records"].count), np.minimum(cnt, cap).astype(np.int32)) and cnt.min() >= 3
    for k in range(cap):
        kept = cnt > k
        assert np.array_equal(_np(a["records"].reward_by_agent)[k][kept], np.stack([want_rec[k], want_rec[k]], 1)[kept]), k


# ------------------------------------------------------------------------------------------------ the rollouts


def _oracle_rewards(env, b, H, f):
    """Each transition of the batch replayed by the oracle without auto-reset from b.states[t] with b.actions[t]:
    sparse + f * float32(phi(s') - phi(s)), [T, N]."""
    T, N = b.dones.shape
    st, ac = _np(b.states), _np(b.actions)
    out = np.zeros((T, N), np.float32)
    for t in range(T):
        ref = st[t].copy()
        sp, _, _, _ = cpu.step(env._tab_host, env._starts_host, ref, ac[t].reshape(N, 2), horizon=H, flags=0)
        dense = (_phi(env, ref) - _phi(env, st[t])).astype(np.float32)
        out[t] = sp.astype(np.float32) + np.float32(f) * dense
    return out


MODES = ["fused", "library", "lstm", "bc", "mixture"]


@pytest.mark.parametrize("mode", MODES)
def test_selfplay_collect_with_phi(mode):
    """collect() with use_phi, graph and eager: everything but the rewards and what follows from them equals the same
    seed's rollout without use_phi; the rewards equal the oracle replay and BatchedOvercookedMultiAgent(use_phi=True)."""
    layout, W, Hh = ("asymmetric_advantages", 9, 5) if mode == "library" else ("cramped_room", 5, 4)
    n, H, T, f, seed = 300, 13, 30, 0.75, 5
    torch.manual_seed(3)
    model = (RllibLSTMShapedCNN if mode == "lstm" else RllibShapedCNN)(W, Hh).cuda()
    partner = {"bc": BCPolicy().cuda(), "mixture": RllibShapedCNN(W, Hh).cuda()}.get(mode)
    envs = [BatchedOvercookedEnv(layout, n, horizon=H, auto_reset=True) for _ in range(3)]
    sps = [SelfPlayRollout(e, model=model, use_graph=g, seed=seed, reward_shaping_factor=f, use_phi=phi,
                           **({} if partner is None else dict(partner=copy.deepcopy(partner), bc_factor=0.5)))
           for e, g, phi in zip(envs[:3], (True, False, True), (True, True, False))]
    sp, sp_eager, sp_plain = sps
    if mode == "fused":
        assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == (True, True, True)
    if mode == "library":
        assert not (sp.fused_first_layer or sp.fused_wide or sp.fused_tail)
    b = sp.collect(T, GAMMA, LAM, keep_logits=True)
    be = sp_eager.collect(T, GAMMA, LAM, keep_logits=True)
    bp = sp_plain.collect(T, GAMMA, LAM, keep_logits=True)
    keys = ["states", "actions", "logp", "values", "rewards", "dones", "last_values", "advantages", "value_targets", "logits"]
    keys += ["state_h", "state_c"] if mode == "lstm" else []
    keys += ["partner_seat"] if partner is not None else []
    for k in keys:
        assert torch.equal(getattr(be, k), getattr(b, k)), k
        if k not in ("rewards", "advantages", "value_targets"):
            assert torch.equal(getattr(bp, k), getattr(b, k)), k
    assert torch.equal(envs[0].state, envs[1].state) and torch.equal(envs[0].state, envs[2].state)
    assert torch.equal(sp.ret_mixed, sp_eager.ret_mixed) and torch.equal(sp.ret_sparse, sp_plain.ret_sparse)
    assert b.dones.any() and not torch.equal(b.rewards, bp.rewards)
    fin, fin_plain = b.episodes.finished(), bp.episodes.finished()
    for k in fin:
        if k != "ep_reward_by_agent":
            assert torch.equal(fin[k], fin_plain[k]), k
    want = _oracle_rewards(envs[0], b, H, f)
    rw = _np(b.rewards).reshape(T, n, 2)
    assert np.array_equal(rw[..., 0], want) and np.array_equal(rw[..., 1], want)
    # the torch reference wrapper, driven by the batch's actions from the same start state
    ma = BatchedOvercookedMultiAgent(BatchedOvercookedEnv(layout, n, horizon=H), reward_shaping_factor=f, use_phi=True)
    ma.reset()
    assert torch.equal(ma.env.state, b.states[0])
    for t in range(T):
        a = b.actions[t].view(n, 2)
        _, r, _, _ = ma.step({"ppo_0": a[:, 0], "ppo_1": a[:, 1]})
        assert torch.equal(r["ppo_0"], b.rewards[t].view(n, 2)[:, 0]) and torch.equal(r["ppo_1"], b.rewards[t].view(n, 2)[:, 1]), t
    adv, tgt = gae_f32(_np(b.rewards), _np(b.values), _np(b.dones), _np(b.last_values), GAMMA, LAM)
    assert np.array_equal(_np(b.advantages), adv) and np.array_equal(_np(b.value_targets), tgt)


def test_selfplay_run_with_phi_keeps_the_restated_returns():
    """run(): ret_mixed and the finished episodes' reward_by_agent are the running sums of the dense rewards."""
    n, H, f = 300, 11, 0.75
    torch.manual_seed(4)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True)
    sp = SelfPlayRollout(env, model=RllibShapedCNN(5, 4).cuda(), seed=2, reward_shaping_factor=f, use_phi=True, episode_capacity=4)
    rm, rw = np.zeros(n, np.float32), np.zeros(n, np.float32)
    recs = [[] for _ in range(n)]
    for t in range(3 * H):
        s = _np(env.state).copy()
        sp.run(1)
        a = _np(sp.actions)
        ref = s.copy()
        sparse, _, done, _ = cpu.step(env._tab_host, env._starts_host, ref, a, horizon=H, flags=0)
        fd = np.float32(f) * (_phi(env, ref) - _phi(env, s)).astype(np.float32)
        r = sparse.astype(np.float32) + fd
        rm = ((rm + sparse.astype(np.float32)) + fd) + fd
        rw = rw + r
        for e in np.nonzero(done)[0]:
            recs[e].append(rw[e])
        rw[done != 0] = 0
        assert np.array_equal(_np(sp.ret_mixed), rm), t
    fin = sp.episodes.finished()
    want = np.array([recs[e][k] for k, e in zip(_slots(fin), _np(fin["env_index"]))], np.float32)
    assert len(want) > n and np.array_equal(_np(fin["ep_reward_by_agent"]), np.stack([want, want], 1))


def _slots(fin):
    """The slot of each row of ``finished()`` (rows are ordered by slot, then environment)."""
    e = _np(fin["env_index"])
    k, seen = np.zeros(len(e), np.int64), {}
    for i, x in enumerate(e):
        k[i] = seen.get(x, 0)
        seen[x] = k[i] + 1
    return k


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pair_collect_with_phi(graph):
    """AgentPairRollout(use_phi=True, random_seats=True): (A, deepcopy(A)) collects SelfPlayRollout(A, use_phi=True)'s
    window at the learner rows; with a BC partner the learner's rewards are the oracle replay's."""
    torch.manual_seed(6)
    n, H, T, f = 517, 20, 30, 0.75
    A = RllibShapedCNN(5, 4).cuda()
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True)
    e1, e2 = mk(), mk()
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=9, use_graph=graph, use_phi=True, reward_shaping_factor=f)
    pair = AgentPairRollout(e2, (A, copy.deepcopy(A)), seed=9, use_graph=graph, random_seats=True, use_phi=True)
    pair.reward_shaping_factor = f
    for w in range(2):
        bs, bp = sp.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        _check_window(bs, bp, pair, False, with_seats=False)
        assert torch.equal(e1.state, e2.state), w
    # next to a BC agent: PPO_BC's window at the learner rows, whose rewards are the oracle replay's
    e3, e4, bc = mk(), mk(), BCPolicy()
    ppo_bc = SelfPlayRollout(e3, model=copy.deepcopy(A), seed=4, partner=copy.deepcopy(bc), bc_factor=1.0, use_graph=graph, use_phi=True,
                             reward_shaping_factor=f)
    pair = AgentPairRollout(e4, (copy.deepcopy(A), bc), seed=4, random_seats=True, use_graph=graph, use_phi=True)
    pair.reward_shaping_factor = f
    bs, bp = ppo_bc.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
    _check_window(bs, bp, pair, False, with_seats=True)
    want = _oracle_rewards(e3, bs, H, f)
    assert np.array_equal(_np(bp.rewards), want) and np.array_equal(_np(bs.rewards).reshape(T, n, 2)[..., 0], want)


def test_captured_graph_follows_the_factor_and_keeps_gamma_099_tables():
    """Inside the captured graph: a new reward_shaping_factor takes effect between replays, and env.potential(0.9) after
    the capture leaves the replayed rewards at gamma 0.99."""
    n, H, T = 300, 13, 20
    torch.manual_seed(7)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True)
    sp = SelfPlayRollout(env, model=RllibShapedCNN(5, 4).cuda(), seed=3, reward_shaping_factor=1.0, use_phi=True)
    sp.collect(T, GAMMA, LAM)
    graph = sp._collect_graphs[(T, False)][1]
    env.potential(0.9)
    for f in (0.25, 3.0):
        sp.reward_shaping_factor = f
        b = sp.collect(T, GAMMA, LAM)
        assert sp._collect_graphs[(T, False)][1] is graph
        want = _oracle_rewards(env, b, H, f)
        rw = _np(b.rewards).reshape(T, n, 2)
        assert np.array_equal(rw[..., 0], want) and np.array_equal(rw[..., 1], want) and b.dones.any()
