"""Agent pairs on the device: the one-view forms of K7, K8, K11 and the draw bit for bit against their two-view forms at the
joint rows 2 e + p(e), and AgentPairRollout against SelfPlayRollout, PPO_BC, each agent's own evaluation, K10, the float64
CNN and the CPU oracle."""
import copy

import numpy as np
import pytest
import torch

import policy_reference as P
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import (PARTNER_DRAW_SALT, AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN,
                                         SelfPlayRollout)
from helpers import TRACE_FILES, TRACE_IDS, Trace
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GUARD = 64


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _swaps(rng, n):
    return {"none": None, "zeros": torch.zeros(n, dtype=torch.int32, device="cuda"),
            "ones": torch.ones(n, dtype=torch.int32, device="cuda"), "mixed": _dev(rng.randint(0, 3, n), torch.int32)}


def _player(seat, swap, n):
    return np.full(n, seat) if swap is None else seat ^ (_np(swap) != 0).astype(np.int64)


def _played_env(layouts, n, seed, horizon=60):
    rng = np.random.RandomState(seed)
    env = BatchedOvercookedEnv(layouts, n, horizon=horizon, auto_reset=True, env_layout=np.arange(n) % len(layouts),
                               rnd_obj_prob_thresh=0.5, seed=seed)
    a = rng.randint(0, 6, size=(25, n, 2)).astype(np.int32)
    env.rollout(_dev(a, torch.int32))
    return env


@pytest.mark.parametrize("layouts", [["cramped_room"], ["cramped_room", "cramped_room_tomato"], POOL_5X4[:8]],
                         ids=["1", "2", "8"])
def test_k7_view_rows_equal_two_view_rows(layouts):
    """Every CPL (n_out 64 / 128 / 256 -> 2 / 4 / 8 columns per lane), swap absent / all 0 / all 1 / mixed, N not a multiple
    of the warps of a CTA; the output's tail past N stays untouched."""
    rng = np.random.RandomState(1)
    n = 333
    env = _played_env(layouts, n, 3)
    for n_out in (64, 128, 256):
        wt = ((torch.rand((520, n_out), device="cuda") - 0.5) * 0.2).to(torch.bfloat16)
        bias = (torch.rand(n_out, device="cuda") - 0.5) * 0.2
        two = env.encoded_linear(wt, bias, neg_slope=0.2).view(n, 2, n_out)
        for name, swap in _swaps(rng, n).items():
            for seat in (0, 1):
                full = torch.full((n + GUARD, n_out), float("nan"), dtype=torch.bfloat16, device="cuda")
                got = env.encoded_linear_view(wt, bias, seat, swap, out=full[:n], neg_slope=0.2)
                p = torch.from_numpy(_player(seat, swap, n)).cuda()
                want = two[torch.arange(n, device="cuda"), p]
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (n_out, name, seat)
                assert torch.isnan(full[n:].float()).all()


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_k7_view_rows_equal_two_view_rows_on_every_fixture(path):
    """The fixtures' states (held soups, idle / cooking / ready pots, objects on counters) of every layout whose table fits
    shared memory; grids that do not fit are refused by both forms."""
    tr = Trace(path)
    st = tr.data["obs_states"]
    n = len(st)
    W, H = tr.layout.width, tr.layout.height
    env = BatchedOvercookedEnv(tr.layout, n, horizon=400)
    env.state.copy_(torch.from_numpy(st))
    rng = np.random.RandomState(W * 31 + H)
    swap = _dev(rng.randint(0, 2, n), torch.int32)
    for n_out in (64, 512):
        wt = _dev(rng.uniform(-0.05, 0.05, size=(W * H * 26, n_out)), torch.bfloat16)
        bias = _dev(rng.uniform(-0.1, 0.1, size=n_out), torch.float32)
        if W * H * 19 * 64 * 2 > 226 * 1024:
            for seat in (0, 1):
                with pytest.raises(RuntimeError, match="shared memory"):
                    env.encoded_linear_view(wt, bias, seat, swap)
            continue
        two = env.encoded_linear(wt, bias, neg_slope=0.2).view(n, 2, n_out)
        for seat in (0, 1):
            got = env.encoded_linear_view(wt, bias, seat, swap, neg_slope=0.2)
            want = two[torch.arange(n, device="cuda"), (swap.long() ^ seat)]
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (n_out, seat)


def _k8(x, tables, counter, seed, actions, values, scores, logp, swap=None, seat=None):
    w1, b1, wh, bh, wo, bo = tables
    args = (x.data_ptr(), x.shape[0], x.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0],
            wo.data_ptr(), bo.data_ptr(), 0.3, 6, seed, counter.data_ptr())
    lib = _native.lib()
    if seat is None:
        _native.check(lib.ovc_policy_tail_logp(*args, actions.data_ptr(), values.data_ptr(), scores.data_ptr(), logp.data_ptr(), None))
    else:
        _native.check(lib.ovc_policy_tail_view(*args, 0 if swap is None else swap.data_ptr(), seat, actions.data_ptr(), values.data_ptr(),
                                               scores.data_ptr(), logp.data_ptr(), None))


@pytest.mark.parametrize("n", [1, 17, 1000])
def test_k8_view_equals_two_view_at_joint_rows(n):
    """Certified-exact dyadic operands (k0 = 160, two hidden layers); the step crosses 2^32; the other seat's actions and
    the outputs' tails are untouched; input rows past N are NaN."""
    rng = np.random.RandomState(n)
    k0 = 160
    x, *w = P.k8_operands(rng, n, k0, 2)
    x, _, _ = P.certified_rows(rng, x, lambda r, m: P.k8_rows(r, m, k0), lambda x: P.k8_reference(x, *w, 0.2, 0.3))
    tables = [_dev(t, torch.bfloat16 if i % 2 == 0 else torch.float32) for i, t in enumerate(w)]
    seed = 0xABCDEF0123
    for name, swap in _swaps(rng, n).items():
        for seat in (0, 1):
            p = _player(seat, swap, n)
            g = 2 * np.arange(n) + p
            x2 = P.k8_rows(rng, 2 * n, k0)
            x2[g] = x
            X2 = _dev(x2, torch.bfloat16)
            xv = torch.full((n + GUARD, k0), float("nan"), dtype=torch.bfloat16, device="cuda")
            xv[:n] = _dev(x, torch.bfloat16)
            c2 = torch.tensor([2**32 - 1, 0], dtype=torch.int64, device="cuda")
            cv = c2.clone()
            for step in range(2):
                a2 = torch.full((2 * n,), 77, dtype=torch.int32, device="cuda")
                v2, lp2 = (torch.zeros(2 * n, device="cuda") for _ in range(2))
                s2 = torch.zeros((2 * n, 8), device="cuda")
                _k8(X2, tables, c2, seed, a2, v2, s2, lp2)
                av = torch.full((n + GUARD, 2), 77, dtype=torch.int32, device="cuda")
                vv, lpv = (torch.full((n + GUARD,), -5.0, device="cuda") for _ in range(2))
                sv = torch.full((n + GUARD, 8), -5.0, device="cuda")
                _k8(xv[:n], tables, cv, seed, av, vv, sv, lpv, swap, seat)
                gi = torch.from_numpy(g).cuda()
                assert torch.equal(av.view(-1)[gi], a2[gi]), (name, seat, step)
                assert (av[:n].view(-1)[torch.from_numpy(2 * np.arange(n) + 1 - p).cuda()] == 77).all() and (av[n:] == 77).all()
                assert torch.equal(vv[:n], v2[gi]) and torch.equal(lpv[:n], lp2[gi]) and torch.equal(sv[:n], s2[gi])
                assert (vv[n:] == -5).all() and (lpv[n:] == -5).all() and (sv[n:] == -5).all()
                P.check_draw(_np(a2), _np(s2), seed, 2**32 - 1 + step)
            assert torch.equal(c2, cv) and int(cv[0]) == 2**32 + 1


def _k11(x, h, c, reset, tables, counter, seed, h_out, c_out, snap, actions, values, logp, scores, swap=None, seat=None):
    w, b, wo, bo = tables
    ptr = lambda t: 0 if t is None else t.data_ptr()
    head = (x.data_ptr(), h.data_ptr(), c.data_ptr(), ptr(reset), x.shape[0], w.data_ptr(), b.data_ptr(), wo.data_ptr(), bo.data_ptr(), 6,
            seed, counter.data_ptr())
    tail = (h_out.data_ptr(), c_out.data_ptr(), ptr(snap[0]), ptr(snap[1]), actions.data_ptr(), values.data_ptr(), logp.data_ptr(),
            scores.data_ptr(), None)
    lib = _native.lib()
    if seat is None:
        _native.check(lib.ovc_lstm_head(*head, *tail))
    else:
        _native.check(lib.ovc_lstm_head_view(*head, ptr(swap), seat, *tail))


@pytest.mark.parametrize("n", [5, 193, 700])
def test_k11_view_equals_two_view_at_joint_rows(n):
    """Per-environment resets, the update in place (view) against out of place (two-view), snapshots, the step across 2^32,
    the other seat's actions untouched."""
    rng = np.random.RandomState(n)
    torch.manual_seed(n)
    m = RllibLSTMShapedCNN(5, 4).cuda()
    from overcooked_ai_b200.selfplay import DenseGridPolicy

    tables = DenseGridPolicy(m, 5, 4, pad_to=16).cuda().lstm_tables()
    seed = 77
    for name, swap in _swaps(rng, n).items():
        seat = int(rng.randint(2))
        p = _player(seat, swap, n)
        gi = torch.from_numpy(2 * np.arange(n) + p).cuda()
        x2 = (torch.randn((2 * n, 64), device="cuda") * 0.5).to(torch.bfloat16)
        h2 = (torch.randn((2 * n, 256), device="cuda") * 0.5).to(torch.bfloat16)
        c2 = torch.randn((2 * n, 256), device="cuda")
        reset = _dev(rng.rand(n) < 0.3, torch.int32)
        xv, hv, cv = x2[gi].contiguous(), h2[gi].contiguous(), c2[gi].contiguous()
        cnt2 = torch.tensor([2**32 - 1, 0], dtype=torch.int64, device="cuda")
        cntv = cnt2.clone()
        for step in range(2):
            ho2, co2 = torch.empty_like(h2), torch.empty_like(c2)
            sh2, sc2 = torch.empty_like(h2), torch.empty_like(c2)
            a2 = torch.full((2 * n,), 77, dtype=torch.int32, device="cuda")
            v2, lp2 = torch.zeros(2 * n, device="cuda"), torch.zeros(2 * n, device="cuda")
            s2 = torch.zeros((2 * n, 8), device="cuda")
            _k11(x2, h2, c2, reset, tables, cnt2, seed, ho2, co2, (sh2, sc2), a2, v2, lp2, s2)
            shv, scv = torch.empty_like(hv), torch.empty_like(cv)
            av = torch.full((n, 2), 77, dtype=torch.int32, device="cuda")
            vv, lpv = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
            sv = torch.zeros((n, 8), device="cuda")
            _k11(xv, hv, cv, reset, tables, cntv, seed, hv, cv, (shv, scv), av, vv, lpv, sv, swap, seat)  # in place
            assert torch.equal(av.view(-1)[gi], a2[gi]), (name, step)
            other = torch.from_numpy(2 * np.arange(n) + 1 - p).cuda()
            assert (av.view(-1)[other] == 77).all()
            assert torch.equal(vv, v2[gi]) and torch.equal(lpv, lp2[gi]) and torch.equal(sv, s2[gi])
            assert torch.equal(hv, ho2[gi]) and torch.equal(cv, co2[gi]) and torch.equal(shv, sh2[gi]) and torch.equal(scv, sc2[gi])
            h2, c2 = ho2, co2
            reset = _dev(rng.rand(n) < 0.3, torch.int32)
        assert torch.equal(cnt2, cntv)


def test_draw_view_matches_philox_at_joint_rows():
    rng = np.random.RandomState(4)
    n, seed = 3001, 0x1234
    env = BatchedOvercookedEnv("cramped_room", n, horizon=50, auto_reset=True)
    scores = _dev(rng.randn(n, 8) * 2, torch.float32)
    for name, swap in _swaps(rng, n).items():
        for seat in (0, 1):
            p = _player(seat, swap, n)
            g = 2 * np.arange(n) + p
            counter = torch.tensor([2**32 - 1, 0], dtype=torch.int64, device="cuda")
            for step in range(2):
                out = torch.full((n, 2), 77, dtype=torch.int32, device="cuda")
                logp = torch.zeros(n, device="cuda")
                env.sample_actions_view(scores, counter, seat, swap, seed=seed, out=out, logp_out=logp)
                full = np.zeros((2 * n, 8), np.float32)
                full[g] = _np(scores)
                v = P.gumbel_scores(full, seed, 2**32 - 1 + step)[g]
                got = _np(out).reshape(-1)
                top2 = np.sort(v, 1)[:, -2:]
                clear = top2[:, 1] - top2[:, 0] > 1e-4
                assert clear.mean() > 0.995 and np.array_equal(got[g][clear], v.argmax(1)[clear]), (name, seat)
                assert (got[2 * np.arange(n) + 1 - p] == 77).all()
                P.check_logp(_np(logp), _np(scores), got[g], 6)
                # bit for bit the two-view draw kernel on the same rows
                c2 = torch.tensor([2**32 - 1 + step, 0], dtype=torch.int64, device="cuda")
                a2 = torch.zeros(2 * n, dtype=torch.int32, device="cuda")
                _native.check(_native.lib().ovc_sample_actions(_dev(full, torch.float32).data_ptr(), 8, 6, 2 * n, seed, c2.data_ptr(),
                                                               a2.data_ptr(), None))
                assert np.array_equal(got[g], _np(a2)[g])


def _records(r):
    fin = r.episodes.finished()
    return {k: _np(v) for k, v in fin.items() if k != "partner_seat"}


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pair_of_one_model_equals_selfplay(lstm, graph):
    """(A, A) == SelfPlayRollout(A) bit for bit on cramped_room over two episodes: K7 -> K9 -> K8 (or -> K8 hidden -> K11)
    on N rows per agent against 2N rows."""
    n, horizon = 517, 20
    torch.manual_seed(3)
    A = RllibLSTMShapedCNN(5, 4) if lstm else RllibShapedCNN(5, 4)
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=9, use_graph=graph, episode_capacity=2)
    pair = AgentPairRollout(e2, (A, A), seed=9, use_graph=graph, episode_capacity=2)
    assert all(a.fused_first_layer and a.fused_wide and a.fused_tail for a in pair.agents)
    for t in range(2 * horizon):
        sp.run(1), pair.run(1)
        assert torch.equal(sp.actions, pair.actions), t
        assert torch.equal(e1.state, e2.state), t
    for k, v in _records(sp).items():
        assert np.array_equal(v, _records(pair)[k]), k
    assert (_np(pair.episodes.finished()["partner_seat"]) == 1).all() and len(_records(pair)["ep_length"]) == 2 * n


def test_pair_with_bc_equals_ppo_bc_over_the_first_episode():
    n, horizon = 640, 25
    torch.manual_seed(5)
    A, bc = RllibShapedCNN(5, 4), BCPolicy()
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=4, partner=copy.deepcopy(bc), bc_factor=1.0, use_graph=False)
    seat = sp.partner_seat.clone()
    assert (seat >= 0).all() and 0 < int(seat.sum()) < n
    swap = (1 - seat).to(torch.int32).contiguous()  # agent 1 (the BC agent) sits at player 1 ^ swap = the partner's seat
    pair = AgentPairRollout(e2, (A, bc), swap=swap, seed=4)
    for t in range(horizon):
        sp.run(1), pair.run(1)
        assert torch.equal(sp.actions, pair.actions), t
        assert torch.equal(e1.state, e2.state), t
    fs, fp = sp.episodes.finished(), pair.episodes.finished()
    for k in fs:
        assert torch.equal(fs[k], fp[k]), k


def test_two_different_agents_act_as_their_own_policies_and_follow_the_oracle():
    """A != B with mixed seats: each agent's actions are its own two-view evaluation of the state at rows 2 e + p(e), with
    the same counter; (bc0, bc1) gives each seat's K10 draw; the environments follow the oracle."""
    rng = np.random.RandomState(8)
    n, horizon, T = 400, 15, 20
    torch.manual_seed(8)
    A, B = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    swap = _dev(rng.randint(0, 2, n), torch.int32)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    shadow = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    pair = AgentPairRollout(env, (A, B), swap=swap, seed=2, use_graph=False)
    own = [SelfPlayRollout(shadow, model=m, seed=2, use_graph=False) for m in (A, B)]
    ar = torch.arange(n, device="cuda")
    st = _np(env.state).copy()
    for t in range(T):
        shadow.state.copy_(env.state)
        for k, sp in enumerate(own):
            sp._draw_counter.copy_(pair.agents[k]._counter)
            sp._policy()
        pair.run(1)
        for k, sp in enumerate(own):
            p = (swap.long() ^ k)
            assert torch.equal(pair.actions[ar, p], sp.actions[ar, p]), (t, k)
        cpu.step(env._tab_host, env._starts_host, st, _np(pair.actions), horizon=horizon, flags=1)
        assert np.array_equal(_np(env.state), st), t
    bc0, bc1 = BCPolicy().cuda(), BCPolicy().cuda()
    env2 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    env2.state.copy_(env.state)
    pair = AgentPairRollout(env2, (bc0, bc1), swap=swap, seed=6, use_graph=False)
    want = torch.full((n, 2), 77, dtype=torch.int32, device="cuda")
    for k, bc in enumerate((bc0, bc1)):
        env.partner_actions(bc.tables(), (swap ^ k).contiguous(), torch.zeros(2, dtype=torch.int64, device="cuda"),
                            seed=6 ^ PARTNER_DRAW_SALT, out=want)
    pair.run(1)
    assert torch.equal(pair.actions, want)


def test_library_path_heads_equal_the_float64_cnn_and_follow_the_oracle():
    """9x5 (no K7 / K9 / K8): K2, the dense model on each agent's rows, the one-view draw.  With exact operands the heads
    equal the float64 CNN on the oracle's encoding of each agent's own view."""
    rng = np.random.RandomState(2)
    n, horizon = 300, 30
    A, B = P.exact_cnn(9, 5, 1), P.exact_cnn(9, 5, 2)
    env = BatchedOvercookedEnv("asymmetric_advantages", n, horizon=horizon, auto_reset=True)
    swap = _dev(rng.randint(0, 2, n), torch.int32)
    pair = AgentPairRollout(env, (A, B), swap=swap, seed=3, use_graph=False)
    assert not any(a.fused_first_layer or a.fused_tail for a in pair.agents)
    st = _np(env.state).copy()
    for t in range(12):
        obs = cpu.encode_lossless(env._tab_host, st, 9, 5, horizon=horizon)
        pair.run(1)
        for k, (m, agent) in enumerate(zip((A, B), pair.agents)):
            logits, value = P.cnn_forward64(m, obs)
            p = _np(swap) ^ k
            g = 2 * np.arange(n) + p
            assert np.array_equal(_np(agent._scores).astype(np.float64), logits[g]), (t, k)
            assert np.array_equal(_np(agent.values).astype(np.float64), value[g]), (t, k)
        cpu.step(env._tab_host, env._starts_host, st, _np(pair.actions), horizon=horizon, flags=1)
        assert np.array_equal(_np(env.state), st), t


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
def test_sync_weights_reaches_the_captured_graph(lstm):
    n = 300
    torch.manual_seed(11)
    mk = (lambda: RllibLSTMShapedCNN(5, 4)) if lstm else (lambda: RllibShapedCNN(5, 4))
    A, bc = mk(), BCPolicy()
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=20, auto_reset=True)
    pair = AgentPairRollout(e1, (A, bc), seed=1)
    pair.run(2)  # captured with the old weights
    with torch.no_grad():
        for q in list(A.parameters()) + list(bc.parameters()):
            q.add_(torch.randn_like(q) * 0.05)
    pair.sync_weights()
    e1.reset()
    if lstm:
        pair.reset_state()
    for a in pair.agents:
        a._counter.zero_()
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=20, auto_reset=True)
    fresh = AgentPairRollout(e2, (copy.deepcopy(A), copy.deepcopy(bc)), seed=1, use_graph=False)
    for t in range(6):
        pair.run(1), fresh.run(1)
        assert torch.equal(pair.actions, fresh.actions), t
        assert torch.equal(e1.state, e2.state), t


def _exact_wide(W, H, seed, hidden=128):
    """P.exact_cnn's function in an RllibShapedCNN with dense layers of ``hidden``: the exact CNN's weights in the first 64
    units, zeros elsewhere.  K7 and K9 fit on 5x4, K8 does not (its layers are 64 wide): K7 -> library layers -> the draw."""
    e = P.exact_cnn(W, H, seed)
    m = RllibShapedCNN(W, H, hidden=hidden).eval()
    with torch.no_grad():
        for name in ("conv_initial", "conv_0", "conv_1"):
            getattr(m, name).load_state_dict(getattr(e, name).state_dict())
        for d, de in zip(list(m.dense) + [m.logits, m.value], list(e.dense) + [e.logits, e.value]):
            d.weight.zero_(), d.bias.zero_()
            d.weight[:de.weight.shape[0], :de.weight.shape[1]].copy_(de.weight), d.bias[:de.bias.shape[0]].copy_(de.bias)
    return m


def test_k7_only_agent_acts_as_its_own_two_view_evaluation():
    """An agent with K7 but not K8 (dense layers of 128) next to a fully fused one, mixed seats: its heads equal the float64
    CNN and its actions its own two-view evaluation (K7 -> library layers -> the draw kernel on 2N rows) at rows 2 e + p(e)
    with the same counter; the environments follow the oracle."""
    rng = np.random.RandomState(12)
    n, horizon, T = 300, 15, 20
    K, A = _exact_wide(5, 4, 3), RllibShapedCNN(5, 4)
    swap = _dev(rng.randint(0, 2, n), torch.int32)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    shadow = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    pair = AgentPairRollout(env, (K, A), swap=swap, seed=2, use_graph=False)
    k = pair.agents[0]
    assert k.fused_first_layer and not k.fused_tail and not k.fused_wide and pair.obs is None
    own = SelfPlayRollout(shadow, model=K, seed=2, use_graph=False)
    assert own.fused_first_layer and not own.fused_tail
    ar, p = torch.arange(n, device="cuda"), swap.long()
    st = _np(env.state).copy()
    for t in range(T):
        shadow.state.copy_(env.state)
        own._draw_counter.copy_(k._counter)
        scores = own._policy()
        shadow.sample_actions(scores, own._draw_counter, seed=2, out=own.actions)
        obs = cpu.encode_lossless(env._tab_host, st, 5, 4, horizon=horizon)
        pair.run(1)
        assert torch.equal(pair.actions[ar, p], own.actions[ar, p]), t
        assert torch.equal(k._scores, scores.view(n, 2, -1)[ar, p]) and torch.equal(k.values, own.values[ar, p]), t
        logits, value = P.cnn_forward64(K, obs)
        g = 2 * np.arange(n) + _np(swap)
        assert np.array_equal(_np(k._scores).astype(np.float64), logits[g]) and np.array_equal(_np(k.values).astype(np.float64), value[g])
        cpu.step(env._tab_host, env._starts_host, st, _np(pair.actions), horizon=horizon, flags=1)
        assert np.array_equal(_np(env.state), st), t


def _exact_lstm(W, H, seed):
    """An RllibLSTMShapedCNN whose convolutions and dense layers are P.exact_cnn's: the LSTM's input is integers (exact in
    any summation order), so the library layers give the same bits on N rows as on 2N; the LSTM's input weights are scaled
    to the input's range."""
    e = P.exact_cnn(W, H, seed)
    torch.manual_seed(seed)
    m = RllibLSTMShapedCNN(W, H).eval()
    with torch.no_grad():
        for name in ("conv_initial", "conv_0", "conv_1"):
            getattr(m, name).load_state_dict(getattr(e, name).state_dict())
        for d, de in zip(m.dense, e.dense):
            d.load_state_dict(de.state_dict())
        m.lstm.weight_ih.mul_(1.0 / 64)
    return m


def test_lstm_pair_on_the_library_path_equals_selfplay():
    """9x5 (no K7 / K8): K2 once per transition for both agents, the dense model on each agent's rows, one-view K11.
    (L, L) equals SelfPlayRollout(L) (library layers on 2N rows, two-view K11) bit for bit over two episodes, with the
    per-environment resets; the environments follow the oracle."""
    n, horizon = 257, 10
    L = _exact_lstm(9, 5, 4)
    e1 = BatchedOvercookedEnv("asymmetric_advantages", n, horizon=horizon, auto_reset=True)
    e2 = BatchedOvercookedEnv("asymmetric_advantages", n, horizon=horizon, auto_reset=True)
    sp = SelfPlayRollout(e1, model=copy.deepcopy(L), seed=6, use_graph=False)
    pair = AgentPairRollout(e2, (L, L), seed=6, use_graph=False)
    assert pair.obs is not None and all(a.lstm and not a.fused_first_layer and not a.fused_tail for a in pair.agents)
    assert all(a.obs is pair.obs for a in pair.agents)
    st = _np(e2.state).copy()
    for t in range(2 * horizon):
        sp.run(1), pair.run(1)
        assert torch.equal(sp.actions, pair.actions), t
        assert torch.equal(sp.values, torch.stack([a.values for a in pair.agents], 1)), t
        for k, a in enumerate(pair.agents):
            assert torch.equal(a.h, sp.h.view(n, 2, -1)[:, k]) and torch.equal(a.c, sp.c.view(n, 2, -1)[:, k]), t
        cpu.step(e2._tab_host, e2._starts_host, st, _np(pair.actions), horizon=horizon, flags=1)
        assert np.array_equal(_np(e2.state), st), t
