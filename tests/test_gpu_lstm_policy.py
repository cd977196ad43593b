"""The LSTM PPO policy on the device: K11 (ovc_lstm_head) on operands whose gate accumulations are certified exact,
K8's hidden output (ovc_policy_hidden) bit for bit, and SelfPlayRollout with RllibLSTMShapedCNN: graph == eager,
run() == collect(), the sequence states of the sample batch replay the learner's forward_sequence, the bootstrap leaves
the live state alone, sync_weights reaches the captured graph, a BC partner, and the environments follow the oracle."""
import copy

import numpy as np
import pytest
import torch

import policy_reference as P
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import PARTNER_DRAW_SALT, BCPolicy, RllibLSTMShapedCNN, SelfPlayRollout, lstm_gate_permutation

pytestmark = pytest.mark.gpu

GUARD = 64
CELL = 256


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _guarded(n, dt, fill, inner=()):
    full = torch.full((n + GUARD,) + tuple(inner), fill, dtype=dt, device="cuda")
    return full[:n], full


def _untouched(full, n, fill):
    tail = full[n:]
    return bool(torch.isnan(tail.float()).all()) if isinstance(fill, float) and np.isnan(fill) else bool((tail == fill).all())


def _sig(z):
    return 1 / (1 + np.exp(-z))


# ----------------------------------------------------------------------------------------------------------------- K11
def _k11_operands(rng, n_rows):
    """x, h_in (bf16-exact dyadic), c_in, w (sparse dyadic, gate rows in kernel order), b, w_heads, b_heads.  Gate
    pre-activations stay within a few units so that sigmoid / tanh are not saturated."""
    x = P.dyadic(rng, (n_rows, 64), 15, [4], density=0.5)
    h = P.dyadic(rng, (n_rows, CELL), 127, [7], density=0.5)
    c = rng.normal(size=(n_rows, CELL)).astype(np.float32).astype(np.float64)
    w = P.dyadic(rng, (4 * CELL, 64 + CELL), 7, [2, 3], density=12 / 320)
    b = P.dyadic(rng, 4 * CELL, 15, [4])
    wo = P.dyadic(rng, (8, CELL), 7, [2, 3], density=0.3)
    bo = P.dyadic(rng, 8, 15, [4])
    return x, h, c, w, b, wo, bo


K11_CASES = [  # (n_rows, n_actions, reset, in_place)
    (1, 6, None, False), (15, 1, "none", True), (17, 7, "all", False), (129, 3, "mixed", True), (1000, 6, "mixed", False),
    (132 * 192 * 2 + 37, 5, "mixed", True),  # 192-row tiles: some CTAs walk three
    (4099, 2, None, True), (255, 4, "all", True),
]


@pytest.mark.parametrize("n_rows,n_actions,reset,in_place", K11_CASES)
def test_k11_exact(n_rows, n_actions, reset, in_place):
    _k11_check(n_rows, n_actions, reset, in_place)


@pytest.mark.parametrize("n_rows,n_actions,reset,in_place", K11_CASES)
def test_k11_view_exact(n_rows, n_actions, reset, in_place):
    """ovc_lstm_head_view: row r is one agent's row of environment r, reset by reset[r], drawn on its joint row
    2 r + seat ^ (swap[r] != 0) (actions [2 n_rows]: the other seat untouched); the state and the other outputs at r."""
    _k11_check(n_rows, n_actions, reset, in_place, seat=n_rows % 2)


def _k11_check(n_rows, n_actions, reset, in_place, seat=None):
    rng = np.random.RandomState(n_rows + 7 * n_actions)
    x, h, c, w, b, wo, bo = _k11_operands(rng, n_rows)
    n_envs = (n_rows + 1) // 2 if seat is None else n_rows
    rs = {None: None, "none": np.zeros(n_envs), "all": np.ones(n_envs), "mixed": rng.rand(n_envs) < 0.4}[reset]
    zero = np.zeros(n_rows, bool) if rs is None else (rs != 0 if seat is not None else np.repeat(rs != 0, 2)[:n_rows])
    swap = None if seat is None or n_rows % 3 == 0 else rng.randint(0, 3, size=n_rows).astype(np.int32)
    r = np.arange(n_rows)
    d = r if seat is None else 2 * r + (seat ^ (0 if swap is None else (swap != 0).astype(np.int64)))
    hu, cu = np.where(zero[:, None], 0, h), np.where(zero[:, None], 0, c)
    z, cert = P.linear(np.concatenate([x, hu], 1), w, b)
    assert cert.holds(), "premise: the gate accumulations are not exact in float32"
    i, f, g, o = (z[:, perm_block] for perm_block in _gate_columns())
    want_c = _sig(f) * cu + _sig(i) * np.tanh(g)
    want_h = _sig(o) * np.tanh(want_c)

    tx, fx = _guarded(n_rows, torch.bfloat16, float("nan"), (64,))
    tx.copy_(_dev(x, torch.bfloat16))
    th, fh = _guarded(n_rows, torch.bfloat16, float("nan"), (CELL,))
    th.copy_(_dev(h, torch.bfloat16))
    tc, fc = _guarded(n_rows, torch.float32, float("nan"), (CELL,))
    tc.copy_(_dev(c, torch.float32))
    h_in0, c_in0 = th.clone(), tc.clone()
    if in_place:
        ho, fho, co, fco = th, fh, tc, fc
    else:
        ho, fho = _guarded(n_rows, torch.bfloat16, float("nan"), (CELL,))
        co, fco = _guarded(n_rows, torch.float32, float("nan"), (CELL,))
    sh, fsh = _guarded(n_rows, torch.bfloat16, float("nan"), (CELL,))
    sc_, fsc = _guarded(n_rows, torch.float32, float("nan"), (CELL,))
    acts, fa = _guarded(n_rows if seat is None else 2 * n_rows, torch.int32, -7)
    vals, fv = _guarded(n_rows, torch.float32, float("nan"))
    lp, fl = _guarded(n_rows, torch.float32, float("nan"))
    s8, fs8 = _guarded(n_rows, torch.float32, float("nan"), (8,))
    treset = None if rs is None else _dev(rs.astype(np.int32), torch.int32)
    tw, tb, two, tbo = _dev(w, torch.bfloat16), _dev(b, torch.float32), _dev(wo, torch.bfloat16), _dev(bo, torch.float32)
    seed = 0xABCD + n_rows
    step0 = 2 ** 32 - 1 if n_rows == 129 else 5  # the draw step crossing 2^32
    counter = torch.tensor([step0, 0], dtype=torch.int64, device="cuda")
    head = (tx.data_ptr(), th.data_ptr(), tc.data_ptr(), 0 if treset is None else treset.data_ptr(), n_rows, tw.data_ptr(), tb.data_ptr(),
            two.data_ptr(), tbo.data_ptr(), n_actions, seed, counter.data_ptr())
    tail = (ho.data_ptr(), co.data_ptr(), sh.data_ptr(), sc_.data_ptr(), acts.data_ptr(), vals.data_ptr(), lp.data_ptr(), s8.data_ptr(), 0)
    if seat is None:
        _native.check(_native.lib().ovc_lstm_head(*head, *tail))
    else:
        tswap = None if swap is None else _dev(swap, torch.int32)
        _native.check(_native.lib().ovc_lstm_head_view(*head, 0 if tswap is None else tswap.data_ptr(), seat, *tail))
    torch.cuda.synchronize()
    assert _np(counter).tolist() == [step0 + 1, 0]
    for full, fill in ((fho, float("nan")), (fco, float("nan")), (fsh, float("nan")), (fsc, float("nan")), (fv, float("nan")),
                       (fl, float("nan")), (fs8, float("nan"))):
        assert _untouched(full, n_rows, fill)
    a_all = _np(fa)
    rest = np.ones(len(a_all), bool)
    rest[d] = False
    assert (a_all[rest] == -7).all(), "an action outside the rows' joint rows was written"
    if not in_place:
        assert torch.equal(th, h_in0) and torch.equal(tc, c_in0)
    # snapshots: the state the row used
    assert np.array_equal(_np(sh.float()), hu) and np.array_equal(_np(sc_), cu)
    # c_out within a few float32 ulp of the float64 cell on the exact gates
    got_c = _np(co).astype(np.float64)
    tol_c = 8 * 2.0 ** -24 * (np.abs(_sig(f) * cu) + np.abs(_sig(i) * np.tanh(g))) + 1e-37
    assert (np.abs(got_c - want_c) <= tol_c).all(), np.abs(got_c - want_c).max()
    # h_out: bf16 of the float64 value, except within the tolerance of a rounding boundary (exempt, counted).  The
    # tolerance is c_out's carried through tanh (slope <= 1) and the output gate, plus a few float32 ulp of h itself.
    got_h = _np(ho.float()).astype(np.float64)
    tol_h = _sig(o) * tol_c + 8 * 2.0 ** -24 * np.abs(want_h) + 1e-37
    near = P.bf16(want_h - tol_h) != P.bf16(want_h + tol_h)
    assert np.array_equal(got_h[~near], P.bf16(want_h)[~near]) and near.mean() < 0.05, near.mean()
    lo, hi = P.bf16(want_h - tol_h)[near], P.bf16(want_h + tol_h)[near]  # rounding is monotone
    assert ((got_h[near] >= lo) & (got_h[near] <= hi)).all()
    # heads bit for bit on the kernel's own h_out where the accumulation is certified exact, else within float32 rounding
    s_want, hc = P.linear(got_h, wo, bo)
    s = _np(s8).astype(np.float64)
    ex = hc.exact()
    assert np.array_equal(s[ex], s_want[ex]) and (np.abs(s - s_want) <= 2.0 ** -20 * hc.abs_sum).all()
    assert np.array_equal(_np(vals), _np(s8)[:, n_actions])
    P.check_draw(a_all[d], s, seed, step0, n_actions, rows=d)
    P.check_logp(_np(lp), s, a_all[d], n_actions)


def _gate_columns():
    """Index arrays of gates i, f, g, o (unit order) into the kernel-ordered gate rows."""
    perm = lstm_gate_permutation(CELL).numpy()
    inv = np.empty_like(perm)
    inv[perm] = np.arange(4 * CELL)
    return [inv[q * CELL:(q + 1) * CELL] for q in range(4)]


def test_k11_refuses_bad_arguments():
    lib = _native.lib()
    t = torch.zeros(64, dtype=torch.float32, device="cuda")
    p = t.data_ptr()
    assert lib.ovc_lstm_head(p, p, p, 0, 2, p, p, p, p, 8, 0, p, p, p, 0, 0, p, 0, 0, 0, 0) != 0
    assert b"n_actions" in lib.ovc_last_error()
    assert lib.ovc_lstm_head(0, p, p, 0, 2, p, p, p, p, 6, 0, p, p, p, 0, 0, p, 0, 0, 0, 0) != 0


# ------------------------------------------------------------------------------------------------------ K8 hidden
def _hidden_reference(x, w_first, b_first, w_hidden, b_hidden, in_slope, slope):
    a = P.bf16(P.leaky(np.asarray(x, np.float64), in_slope))
    z, cert = P.linear(a, w_first, b_first)
    certs = [cert]
    a = P.bf16(P.leaky(z, slope))
    for l in range(len(w_hidden)):
        z, cert = P.linear(a, w_hidden[l], b_hidden[l])
        certs.append(cert)
        a = P.bf16(P.leaky(z, slope))
    return a, certs


@pytest.mark.parametrize("k0,n_hidden", [(32 * (i + 1), i if i < 8 else 0) for i in range(8)] + [(160, 8), (256, 0), (64, 2)])
def test_k8_hidden_output_exact(k0, n_hidden):
    n_rows = 4099 if k0 % 64 else 101381
    rng = np.random.RandomState(k0 + n_hidden)
    x, w1, b1, wh, bh, _, _ = P.k8_operands(rng, n_rows, k0, n_hidden)
    in_slope, slope = 0.25, 0.5
    x, want, certs = P.certified_rows(rng, x, lambda r, n: P.k8_rows(r, n, k0), lambda x: _hidden_reference(x, w1, b1, wh, bh, in_slope, slope))
    assert all(c.holds() for c in certs), "premise"
    tx, _ = _guarded(n_rows, torch.bfloat16, float("nan"), (k0,))
    tx.copy_(_dev(x, torch.bfloat16))
    out, full = _guarded(n_rows, torch.bfloat16, float("nan"), (64,))
    whd = _dev(wh if n_hidden else np.zeros((1, 64, 64)), torch.bfloat16)
    bhd = _dev(bh if n_hidden else np.zeros((1, 64)), torch.float32)
    w1d, b1d = _dev(w1, torch.bfloat16), _dev(b1, torch.float32)
    _native.check(_native.lib().ovc_policy_hidden(tx.data_ptr(), n_rows, k0, in_slope, w1d.data_ptr(), b1d.data_ptr(), whd.data_ptr(),
                                                  bhd.data_ptr(), n_hidden, slope, out.data_ptr(), 0))
    got = _np(out.float())
    assert np.array_equal(got, want), (got != want).sum()
    assert _untouched(full, n_rows, float("nan"))


# ---------------------------------------------------------------------------------------------- SelfPlayRollout
LAYOUTS = ["cramped_room", "asymmetric_advantages"]  # K7 -> K9 -> K8 -> K11; K2 + library trunk -> K11


def _rollout(layout, n, horizon, model, use_graph, seed=3, **kw):
    env = BatchedOvercookedEnv(layout, n, horizon=horizon, auto_reset=True)
    return SelfPlayRollout(env, model=model, use_graph=use_graph, seed=seed, **kw)


def _model(layout, seed=0):
    from overcooked_ai_b200 import layout as L

    l = L.compile_layout(layout)
    torch.manual_seed(seed)
    return RllibLSTMShapedCNN(l.width, l.height)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_lstm_rollout_graph_eager_run_collect_and_oracle(layout):
    n, T, H = 300, 23, 9
    model = _model(layout)
    sp_g = _rollout(layout, n, H, model, True, max_seq_len=5)
    sp_e = _rollout(layout, n, H, model, False, max_seq_len=5)
    sp_r = _rollout(layout, n, H, model, False)
    if layout == "cramped_room":
        assert sp_g.fused_first_layer and sp_g.fused_wide and sp_g.fused_tail
    else:
        assert not sp_g.fused_tail
    for w in range(2):  # the second window continues from the live state
        bg, be = sp_g.collect(T, 0.99, 0.95), sp_e.collect(T, 0.99, 0.95)
        for k in ("actions", "logp", "values", "rewards", "dones", "last_values", "advantages", "state_h", "state_c", "states"):
            assert torch.equal(getattr(bg, k), getattr(be, k)), k
        assert torch.equal(sp_g.h, sp_e.h) and torch.equal(sp_g.c, sp_e.c)
        # run() draws what collect() draws, and without the bootstrap ends in the same live state
        ref = _np(sp_r.env.state).copy()
        for t in range(T):
            if t % 5 == 0:  # the batch's sequence state is run()'s live state after the reset rule
                keep = torch.ones(2 * n, dtype=torch.bool, device="cuda") if t == 0 else (be.dones[t - 1] == 0).repeat_interleave(2)
                assert torch.equal(sp_r.h[keep], be.state_h[t // 5][keep]) and torch.equal(sp_r.c[keep], be.state_c[t // 5][keep]), (w, t)
            assert torch.equal(sp_r.env.state, be.states[t]), (w, t)
            sp_r.run(1)
            a, want = _np(sp_r.actions).reshape(-1), _np(be.actions[t])
            assert np.array_equal(a, want), (w, t, (a != want).sum())
            cpu.step(sp_r.env._tab_host, sp_r.env._starts_host, ref, _np(sp_r.actions), horizon=H, flags=1)
            assert np.array_equal(_np(sp_r.env.state), ref), t
        assert torch.equal(sp_r.h, sp_e.h) and torch.equal(sp_r.c, sp_e.c)
    assert bg.dones.any()


HEAD_SCALE = 30.0  # the heads of a fresh model give logits of a few 1e-2; scaled, the LSTM state moves them by O(1)
REPLAY_TOL = 0.015  # |kernel - float64| / (1 + |float64|): bf16 activations at every layer and bf16 h, about 3 bf16 ulp


def _replay_model(layout):
    """A seeded RllibLSTMShapedCNN with its heads scaled by HEAD_SCALE and every weight bf16-representable, so that the
    bf16 policy holds the model's own weights and the remaining difference is the activations' rounding."""
    m = _model(layout, 1)
    with torch.no_grad():
        m.logits.weight.mul_(HEAD_SCALE), m.value.weight.mul_(HEAD_SCALE)
        for p_ in m.parameters():
            p_.copy_(p_.bfloat16().float())
    return m


def _replay_error(ref, b, obs_all, state):
    """max over the window of |kernel - forward_sequence| / (1 + |forward_sequence|) for the heads and values, every chunk k
    replayed from state(k) = (h, c) with reset[t] = dones[t - 1] inside the chunk."""
    T, L = b.dones.shape[0], b.seq_len
    dones = _np(b.dones).astype(bool)
    worst = 0.0
    for k in range(-(-T // L)):
        t0, t1 = k * L, min(T, (k + 1) * L)
        reset = torch.zeros((t1 - t0, obs_all.shape[1]), dtype=torch.uint8)
        for t in range(t0 + 1, t1):
            reset[t - t0] = torch.from_numpy(np.repeat(dones[t - 1], 2).astype(np.uint8))
        h, c = state(k)
        with torch.no_grad():
            lg, v, _ = ref.forward_sequence(obs_all[t0:t1], h, c, reset)
        for got, want in ((b.logits[t0:t1, :, :6], lg), (b.values[t0:t1], v)):
            want = want.numpy()
            worst = max(worst, float((np.abs(_np(got).astype(np.float64) - want) / (1 + np.abs(want))).max()))
    return worst


@pytest.mark.parametrize("layout", LAYOUTS)
def test_lstm_batch_replays_forward_sequence(layout):
    """keep_logits heads / values against forward_sequence in float64 on the re-encoded observations, chunk by chunk from
    state_h / state_c with the dones rule, within REPLAY_TOL; the state is zero at every episode start.  The same replay from
    a zeroed or a unit-permuted state must exceed the tolerance several times over (the comparison can see a wrong state).
    Horizon 7 with chunks of 5: the second window's episodes end inside chunks (the reset rule) and at a chunk's last step
    (the stored state)."""
    n, T, L, H = 64, 20, 5, 7
    model = _replay_model(layout)
    sp = _rollout(layout, n, H, model, True, max_seq_len=L)
    sp.collect(T, 0.99, 0.95, keep_logits=True)  # a first window: the second starts mid-episode with a live state
    b = sp.collect(T, 0.99, 0.95, keep_logits=True)
    assert b.seq_len == L and b.state_h.shape == (-(-T // L), 2 * n, CELL)
    dones = _np(b.dones).astype(bool)
    starts = 0
    for k in range(1, -(-T // L)):  # zero state at every episode start
        ended = np.repeat(dones[k * L - 1], 2)
        starts += int(ended.sum())
        assert (_np(b.state_h[k].float())[ended] == 0).all() and (_np(b.state_c[k])[ended] == 0).all()
    assert starts > 0 and dones[[t for t in range(T) if t % L != L - 1]].any()
    ref = copy.deepcopy(model).double().cpu()
    obs_all = b.observations(torch.arange(T * n, device="cuda")).view(T, n * 2, sp.W, sp.H, 26).permute(0, 1, 4, 2, 3).double().cpu()
    stored = lambda k: (b.state_h[k].double().cpu(), b.state_c[k].double().cpu())
    err = _replay_error(ref, b, obs_all, stored)
    assert err <= REPLAY_TOL, err
    perm = torch.randperm(CELL)
    wrong = {"zero": lambda k: tuple(torch.zeros_like(s) for s in stored(k)),
             "permuted": lambda k: tuple(s[:, perm] for s in stored(k))}
    for name, state in wrong.items():
        e = _replay_error(ref, b, obs_all, state)
        assert e > 4 * REPLAY_TOL, (name, e, err)


def test_lstm_sync_weights_reaches_the_captured_graph():
    """A captured collect() after sync_weights() equals an eager rollout built afresh from the updated model and continued
    from the same environments, live state and draw counter; the K11 tables did change."""
    layout, n, T = "cramped_room", 200, 12
    model_g, model_e = _model(layout, 2), _model(layout, 2)
    sp_g = _rollout(layout, n, 8, model_g, True)
    sp_e = _rollout(layout, n, 8, model_e, False)
    sp_g.collect(T, 0.99, 0.95), sp_e.collect(T, 0.99, 0.95)
    assert torch.equal(sp_g.h, sp_e.h) and torch.equal(sp_g.env.state, sp_e.env.state)
    old = [t.clone() for t in sp_g._lstm_tables]
    for m in (model_g, model_e):
        torch.manual_seed(9)
        with torch.no_grad():
            for p_ in m.parameters():
                p_.add_(torch.randn_like(p_) * 0.05)
    sp_g.sync_weights()
    assert not any(torch.equal(a, b) for a, b in zip(old, sp_g._lstm_tables))
    fresh = SelfPlayRollout(sp_e.env, model=model_e, use_graph=False, seed=3)  # folds the updated model, no sync_weights
    fresh.h.copy_(sp_e.h), fresh.c.copy_(sp_e.c), fresh._draw_counter.copy_(sp_e._draw_counter)
    bg, bf = sp_g.collect(T, 0.99, 0.95), fresh.collect(T, 0.99, 0.95)
    for k in ("actions", "logp", "values", "last_values", "state_h", "state_c", "states"):
        assert torch.equal(getattr(bg, k), getattr(bf, k)), k


def test_lstm_collect_with_a_bc_partner():
    """bc_factor = 1: every environment has the partner.  At t = 0 the learner's rows draw what a rollout without the partner
    draws (same model, seed and start state), and the partner's rows are K10's draw on the same state."""
    layout, n, T = "cramped_room", 200, 12
    model = _model(layout, 3)
    bc = BCPolicy()
    sp_p = _rollout(layout, n, 8, model, True, partner=bc, bc_factor=1.0)
    sp_0 = _rollout(layout, n, 8, model, False)
    b, b0 = sp_p.collect(T, 0.99, 0.95), sp_0.collect(T, 0.99, 0.95)
    seat = b.partner_seat[0].long()
    assert (seat >= 0).all() and torch.equal(b.states[0], b0.states[0])
    env = BatchedOvercookedEnv(layout, n, horizon=8, auto_reset=True)
    assert torch.equal(env.state, b.states[0])
    want = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    env.partner_actions(bc.to("cuda").tables(), seat.int(), torch.zeros(2, dtype=torch.int64, device="cuda"), seed=3 ^ PARTNER_DRAW_SALT,
                        out=want)
    got, no_partner = b.actions[0].view(n, 2), b0.actions[0].view(n, 2)
    e = torch.arange(n, device="cuda")
    assert torch.equal(got[e, seat], want[e, seat]) and torch.equal(got[e, 1 - seat], no_partner[e, 1 - seat])
    mask = b.learner_mask.view(T, n, 2)
    assert (mask.sum(-1) == 1).all() and torch.isfinite(b.advantages).all()


def test_lstm_policy_refuses_float32():
    env = BatchedOvercookedEnv("cramped_room", 4, horizon=10, auto_reset=True)
    with pytest.raises(AssertionError, match="K11"):
        SelfPlayRollout(env, model=RllibLSTMShapedCNN(5, 4), autocast_dtype=None)
