"""The policy kernels K7 / K9 / K8, the draw kernel and the sample-batch kernels on operands where their float32
arithmetic is exact (tests/policy_reference.py): every output must equal a float64 restatement bit for bit, memory past
every output's end must stay untouched, and the PPO behaviour policy that collect() evaluates must be the learner's
network itself."""
import copy

import numpy as np
import pytest
import torch

import policy_reference as P
from helpers import TRACE_FILES, TRACE_IDS, Trace
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN, SelfPlayRollout
from ppo_reference import gae_f32

pytestmark = pytest.mark.gpu

GUARD = 64  # sentinel elements past each output's end


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _guarded(n, dt, fill, inner=()):
    """(view of the first n rows, whole allocation): the rows past n hold ``fill``."""
    full = torch.full((n + GUARD,) + tuple(inner), fill, dtype=dt, device="cuda")
    return full[:n], full


def _tail_untouched(full, n, fill):
    tail = full[n:]
    if isinstance(fill, float) and np.isnan(fill):
        return bool(torch.isnan(tail.float()).all())
    return bool((tail == fill).all())


# ------------------------------------------------------------------------------------------------------------------ K7
def _k7_check(env, rng, n_out, slope, view_swap=None):
    l = env.layouts[0]
    st = _np(env.state)
    obs = cpu.encode_lossless(env._tab_host, st, l.width, l.height, env.horizon).astype(np.float64)
    if view_swap is not None:
        sw = _np(view_swap) != 0
        obs[sw] = obs[sw][:, ::-1]
    wt, b = P.k7_operands(rng, obs.shape[2] * obs.shape[3] * obs.shape[4], n_out)
    want, certs = P.k7_reference(obs.reshape(2 * len(st), -1), wt, b, slope)
    assert certs[0].holds(), "premise: the operands are not exact in float32"
    out, full = _guarded(2 * len(st), torch.bfloat16, float("nan"), (n_out,))
    env.encoded_linear(_dev(wt, torch.bfloat16), _dev(b, torch.float32), out=out, neg_slope=slope, view_swap=view_swap)
    got = _np(out.float())
    assert np.array_equal(got, want), (n_out, np.abs(got - want).max(), (got != want).sum())
    assert _tail_untouched(full, 2 * len(st), float("nan"))
    return obs


def _k7_fits(l):
    return l.width * l.height * 19 * 64 * 2 <= 226 * 1024


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_k7_exact_on_fixture_states(path):
    tr = Trace(path)
    if not _k7_fits(tr.layout):
        pytest.skip("the table of this grid does not fit shared memory (K7 refuses it)")
    st = tr.data["obs_states"]
    env = BatchedOvercookedEnv(tr.layout, len(st), horizon=400)
    env.state.copy_(torch.from_numpy(st))
    rng = np.random.RandomState(len(st))
    for n_out, slope in ((64, 0.25), (128, 0.0), (512, 0.5)):
        _k7_check(env, rng, n_out, slope)


@pytest.mark.parametrize("layout,n", [("long_cook_time", 777), ("counter_circuit", 1027), ("cramped_room", 2 * 333 + 1)])
def test_k7_exact_on_random_rollouts(layout, n):
    """Random start states (held objects, cooking pots) then random play; every n_out from one to several column slices
    per CTA set; view_swap; the urgency plane exactly at its edge (horizon - t = 40 and 39)."""
    horizon = 60
    env = BatchedOvercookedEnv(layout, n, horizon=horizon, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=n)
    rng = np.random.RandomState(n)
    acts = rng.randint(0, 6, size=(25, n, 2)).astype(np.int32)
    acts[rng.rand(25, n, 2) < 0.4] = 5
    env.rollout(torch.from_numpy(acts).cuda())
    assert _k7_fits(env.layouts[0])
    for n_out in (64, 128, 256, 512, 1024):
        _k7_check(env, rng, n_out, 0.25)
    swap = torch.from_numpy((rng.rand(n) < 0.5).astype(np.int32)).cuda()
    _k7_check(env, rng, 128, 1.0, view_swap=swap)
    st = env.state.clone()
    for t in (horizon - 40, horizon - 39):
        env.state.copy_(st)
        env.state[:, 0] = t
        urgency = _k7_check(env, rng, 256, 0.0)[..., 25]
        assert (urgency == 1).all() if t == horizon - 39 else not urgency.any()


def test_k7_exact_on_several_layouts_per_call():
    """1, 2 and 8 layouts of the 5x4 shape in one call (each with its own terrain and cook times); a 9th is refused."""
    from overcooked_ai_b200 import layout as L

    names = [n for n in L.layout_names() if _compiles(n) and (L.compile_layout(n).width, L.compile_layout(n).height) == (5, 4)]
    assert len(names) >= 9
    rng = np.random.RandomState(9)
    for k, n in ((1, 1), (2, 67), (8, 8 * 129 + 3)):
        env = BatchedOvercookedEnv(names[:k], n, horizon=50, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=k)
        acts = rng.randint(0, 6, size=(12, n, 2)).astype(np.int32)
        env.rollout(torch.from_numpy(acts).cuda())
        assert len(np.unique(env.env_layout_host)) == min(k, n)
        _k7_check(env, rng, 192, 0.25)
    env = BatchedOvercookedEnv(names[:9], 90, horizon=50)
    wt = torch.zeros((520, 64), dtype=torch.bfloat16, device="cuda")
    with pytest.raises(RuntimeError, match="more than 8 layouts"):
        env.encoded_linear(wt, torch.zeros(64, device="cuda"))


def _compiles(name):
    from overcooked_ai_b200 import layout as L

    try:
        L.compile_layout(name)
        return True
    except ValueError:
        return False


# ------------------------------------------------------------------------------------------------------------------ K9
def _k9(a0, m, w1, b1, w2, b2, slope, z2):
    return _native.lib().ovc_wide_layers(a0.data_ptr(), m, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(), 160, slope,
                                         z2.data_ptr(), 0)


@pytest.mark.parametrize("m,slope", [(1, 0.25), (127, 1.0), (128, 0.0), (129, 0.25), (132 * 128 - 1, 1.0), (132 * 128 + 1, 0.0),
                                     (128 * 449 + 5, 0.25)])
def test_k9_exact(m, slope):
    """Partial and full tiles, one tile per SM and one more, several tiles per persistent CTA; a0 rows past m hold NaN
    (the tensor map bounds them) and z2 rows past m stay untouched."""
    rng = np.random.RandomState(m)
    a0, w1, b1, w2, b2 = P.k9_operands(rng, m)
    a0, want, certs = P.certified_rows(rng, a0, P.k9_rows, lambda x: P.k9_reference(x, w1, b1, w2, b2, slope))
    assert all(c.holds() for c in certs), "premise"
    ta0, _ = _guarded(m, torch.bfloat16, float("nan"), (512,))
    ta0.copy_(_dev(a0, torch.bfloat16))
    z2, full = _guarded(m, torch.bfloat16, float("nan"), (160,))
    _native.check(_k9(ta0, m, _dev(w1, torch.bfloat16), _dev(b1, torch.float32), _dev(w2, torch.bfloat16), _dev(b2, torch.float32), slope, z2))
    got = _np(z2.float())
    assert np.array_equal(got, want), ((got != want).sum(), np.abs(got - want).max())
    assert _tail_untouched(full, m, float("nan"))


# ------------------------------------------------------------------------------------------------------------------ K8
def _k8_cases():
    """A covering set: every K0 with n_hidden 0 and 8 and with and without logp; every n_hidden, n_actions, slope pair and
    row count appears.  101 381 rows: every warp of the 132 x 16 walks three tiles."""
    slopes = [(0.0, 0.25), (0.25, 0.5), (0.5, 1.0), (1.0, 0.0)]
    rows = [1, 15, 16, 17, 4099, 101381]
    cases = []
    for i, k0 in enumerate(range(32, 257, 32)):
        for j, nh in enumerate((0, 8)):
            c = len(cases)
            cases.append((k0, nh, 1 + c % 7, slopes[c % 4], rows[c % 5], (i + j) % 2 == 0))
    cases += [(160, 1, 6, (0.25, 0.25), 101381, True), (96, 3, 7, (1.0, 1.0), 4099, False), (224, 3, 3, (0.0, 0.0), 17, True)]
    return cases


def _k8_run(x, ops, n_rows, k0, n_hidden, n_actions, in_slope, slope, seed, counter, logp):
    """K8 with guarded outputs (checked untouched past n_rows); returns (actions, values, scores, logp) of the n_rows rows."""
    w1, b1, wh, bh, wo, bo = ops
    acts, fa = _guarded(n_rows, torch.int32, -7)
    vals, fv = _guarded(n_rows, torch.float32, float("nan"))
    sc, fs = _guarded(n_rows, torch.float32, float("nan"), (8,))
    lp, fl = _guarded(n_rows, torch.float32, float("nan"))
    args = (x.data_ptr(), n_rows, k0, in_slope, w1.data_ptr(), b1.data_ptr(), wh.data_ptr() if n_hidden else 0, bh.data_ptr() if n_hidden else 0,
            n_hidden, wo.data_ptr(), bo.data_ptr(), slope, n_actions, seed, counter.data_ptr(), acts.data_ptr(), vals.data_ptr(),
            sc.data_ptr())
    lib = _native.lib()
    _native.check(lib.ovc_policy_tail_logp(*args, lp.data_ptr(), 0) if logp else lib.ovc_policy_tail(*args, 0))
    assert _tail_untouched(fa, n_rows, -7) and _tail_untouched(fv, n_rows, float("nan"))
    assert _tail_untouched(fs, n_rows, float("nan")) and _tail_untouched(fl, n_rows if logp else 0, float("nan"))
    return _np(acts), _np(vals), _np(sc), _np(lp)


def _k8_device_ops(ops):
    w1, b1, wh, bh, wo, bo = ops
    wh = wh if len(wh) else np.zeros((1, 64, 64))
    bh = bh if len(bh) else np.zeros((1, 64))
    return (_dev(w1, torch.bfloat16), _dev(b1, torch.float32), _dev(wh, torch.bfloat16), _dev(bh, torch.float32), _dev(wo, torch.bfloat16),
            _dev(bo, torch.float32))


@pytest.mark.parametrize("k0,n_hidden,n_actions,slopes,n_rows,logp", _k8_cases())
def test_k8_exact(k0, n_hidden, n_actions, slopes, n_rows, logp):
    """Heads and values bit for bit; actions = the draw on the exact heads; logp within 1e-5 of the float64 log-softmax;
    x rows past n_rows hold NaN and no output past n_rows is written."""
    in_slope, slope = slopes
    rng = np.random.RandomState(k0 * 100 + n_hidden * 10 + n_rows % 7)
    x, *ops = P.k8_operands(rng, n_rows, k0, n_hidden)
    x, heads, certs = P.certified_rows(rng, x, lambda r, n: P.k8_rows(r, n, k0), lambda x: P.k8_reference(x, *ops, in_slope, slope))
    assert all(c.holds() for c in certs), "premise"
    tx, _ = _guarded(n_rows, torch.bfloat16, float("nan"), (k0,))
    tx.copy_(_dev(x, torch.bfloat16))
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    dops = _k8_device_ops(ops)
    for step in range(2):
        a, v, s, lp = _k8_run(tx, dops, n_rows, k0, n_hidden, n_actions, in_slope, slope, 0xC0FFEE + k0, counter, logp)
        assert np.array_equal(s, heads), ((s != heads).sum(), np.abs(s - heads).max())
        assert np.array_equal(v, heads[:, n_actions])
        assert _np(counter).tolist() == [step + 1, 0]
        P.check_draw(a, heads, 0xC0FFEE + k0, step, n_actions)
        if logp:
            P.check_logp(lp, heads, a, n_actions)


# ------------------------------------------------------------------------------------------------ draws past step 2^32
def test_draw_counter_past_2_to_the_32():
    """The step's high word enters Philox word 3 (2 step_hi + block): two launches from step 2^32 - 1 draw at steps
    2^32 - 1 and 2^32, and the counter ends at 2^32 + 1, for ovc_sample_actions[_logp] and K8."""
    lib = _native.lib()
    rng = np.random.RandomState(5)
    n = 4099
    scores = rng.normal(size=(n, 8)) * 2
    tsc = _dev(scores, torch.float32)
    start = 2 ** 32 - 1
    for logp in (False, True):
        counter = torch.tensor([start, 0], dtype=torch.int64, device="cuda")
        for k in range(2):
            acts, fa = _guarded(n, torch.int32, -7)
            lp, fl = _guarded(n, torch.float32, float("nan"))
            if logp:
                _native.check(lib.ovc_sample_actions_logp(tsc.data_ptr(), 8, 7, n, 321, counter.data_ptr(), acts.data_ptr(), lp.data_ptr(), 0))
                P.check_logp(_np(lp), scores, _np(acts), 7)
            else:
                _native.check(lib.ovc_sample_actions(tsc.data_ptr(), 8, 7, n, 321, counter.data_ptr(), acts.data_ptr(), 0))
            P.check_draw(_np(acts), scores, 321, start + k, 7)
            assert _tail_untouched(fa, n, -7) and _tail_untouched(fl, n if logp else 0, float("nan"))
        assert _np(counter).tolist() == [2 ** 32 + 1, 0]
    x, *ops = P.k8_operands(rng, n, 64, 1)
    x, heads, _ = P.certified_rows(rng, x, lambda r, m: P.k8_rows(r, m, 64), lambda x: P.k8_reference(x, *ops, 0.25, 0.5))
    counter = torch.tensor([start, 0], dtype=torch.int64, device="cuda")
    dops = _k8_device_ops(ops)
    for k in range(2):
        a, _, s, lp = _k8_run(_dev(x, torch.bfloat16), dops, n, 64, 1, 6, 0.25, 0.5, 77, counter, True)
        assert np.array_equal(s, heads)
        P.check_draw(a, heads, 77, start + k, 6)
        P.check_logp(lp, heads, a, 6)
    assert _np(counter).tolist() == [2 ** 32 + 1, 0]


# ------------------------------------------------------------------------------------ sample-batch kernels: guards, GAE
def test_sample_batch_kernels_leave_memory_past_their_outputs_alone():
    """ovc_record_transition and ovc_gae write exactly their outputs' rows; GAE input rows past the window hold NaN and
    change nothing; the GAE is bit-exact at window lengths around its 16-step unroll."""
    n = 1001
    env = BatchedOvercookedEnv("cramped_room", n, horizon=9, auto_reset=True)
    rng = np.random.RandomState(3)
    factor = torch.full((1,), 0.5, dtype=torch.float32, device="cuda")
    for t in range(12):
        sp, sh, dn, _ = [_np(x) for x in env.step(_dev(rng.randint(0, 6, size=(n, 2)), torch.int32))]
        rw, frw = _guarded(2 * n, torch.float32, float("nan"))
        dd, fdd = _guarded(n, torch.uint8, 0xA5)
        env.record_transition(factor, rewards=rw, dones=dd)
        assert np.array_equal(_np(rw).reshape(n, 2), sp[:, None] + np.float32(0.5) * sh.astype(np.float32))
        assert np.array_equal(_np(dd), (dn != 0).astype(np.uint8))
        assert _tail_untouched(frw, 2 * n, float("nan")) and _tail_untouched(fdd, n, 0xA5)
    R = 2 * n
    for T in (15, 16, 17, 33):
        r, v = rng.normal(size=(T, R)).astype(np.float32), rng.normal(size=(T, R)).astype(np.float32)
        d = (rng.rand(T, n) < 0.1).astype(np.uint8)
        last = rng.normal(size=R).astype(np.float32)
        ins = []
        for arr, dt, fill in ((r, torch.float32, float("nan")), (v, torch.float32, float("nan")), (d, torch.uint8, 1)):
            full = torch.full((T + 1,) + arr.shape[1:], fill, dtype=dt, device="cuda")
            full[:T].copy_(_dev(arr, dt))
            ins.append(full[:T])
        adv, fadv = _guarded(T, torch.float32, float("nan"), (R,))
        tgt, ftgt = _guarded(T, torch.float32, float("nan"), (R,))
        env.gae(ins[0], ins[1], ins[2], _dev(last, torch.float32), 0.99, 0.95, adv, tgt)
        want_adv, want_tgt = gae_f32(r, v, d, last, 0.99, 0.95)
        assert np.array_equal(_np(adv), want_adv) and np.array_equal(_np(tgt), want_tgt), T
        assert _tail_untouched(fadv, T, float("nan")) and _tail_untouched(ftgt, T, float("nan"))


# ------------------------------------------------------------------------------ end to end: the behaviour policy is the net
def _load(dst, src):
    with torch.no_grad():
        for p, q in zip(dst.parameters(), src.parameters()):
            p.copy_(q)


def _check_batch(b, env, cnn, T):
    """logits / values of every slot == the float64 forward of ``cnn`` on observations() of states[t]; logp to 1e-5."""
    n = env.n_envs
    obs = _np(b.observations(torch.arange(T * n, device="cuda")))
    assert (obs <= P.plane_bounds()).all(), "premise: an observation exceeds the planes' bounds"
    logits, values = P.cnn_forward64(cnn, obs)
    logits, values = logits.reshape(T, 2 * n, 6), values.reshape(T, 2 * n)
    assert np.array_equal(_np(b.logits)[..., :6], logits) and np.array_equal(_np(b.values), values)
    for t in range(T):
        P.check_logp(_np(b.logp[t]), logits[t], _np(b.actions[t]), 6)
    last = env.lossless_state_encoding()
    assert np.array_equal(_np(b.last_values), P.cnn_forward64(cnn, _np(last))[1])
    assert len(np.unique(logits)) > 8 and len(np.unique(_np(b.actions))) == 6


@pytest.mark.parametrize("layout,flags", [("cramped_room", (True, True, True)), ("coordination_ring", (True, False, False)),
                                          ("asymmetric_advantages", (False, False, False))])
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_collect_evaluates_the_learners_network(layout, flags, use_graph):
    """With exact weights the behaviour policy's heads equal the float64 CNN on the batch's own observations, bit for
    bit, through K7 -> K9 -> K8, K7 + library GEMMs and K2 + library GEMMs; after a second weight set with another wiring is
    loaded and sync_weights() called, the next collect (the same captured graph) equals the new network."""
    n, T = 256, 12
    W, H = BatchedOvercookedEnv(layout, 1).layouts[0].width, BatchedOvercookedEnv(layout, 1).layouts[0].height
    model = P.exact_cnn(W, H, seed=11).cuda()
    env = BatchedOvercookedEnv(layout, n, horizon=7, auto_reset=True)
    sp = SelfPlayRollout(env, model=model, use_graph=use_graph, seed=4)
    assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == flags
    b = sp.collect(T, 0.99, 0.95, keep_logits=True)
    _check_batch(b, env, model, T)
    graph = sp._collect_graphs.get((T, True))
    second = P.exact_cnn(W, H, seed=12)
    _load(model, second)
    sp.sync_weights()
    b = sp.collect(T, 0.99, 0.95, keep_logits=True)
    assert sp._collect_graphs.get((T, True)) is graph
    _check_batch(b, env, second, T)


def test_device_fold_is_the_float64_fold():
    """DenseGridPolicy of a CUDA model with full-precision weights == the float64 host fold, to float32 round-off."""
    torch.manual_seed(6)
    for W, H in ((5, 4), (9, 5)):
        cnn = RllibShapedCNN(W, H).eval()
        host = DenseGridPolicy(copy.deepcopy(cnn).double(), W, H, pad_to=16).double()
        dev = DenseGridPolicy(cnn.cuda(), W, H, pad_to=16)
        for (name, p), q in zip(dev.named_parameters(), host.parameters()):
            got, want = p.detach().double().cpu().numpy(), q.detach().numpy()
            assert (np.abs(got - want) <= 1e-6 * np.abs(want)).all(), (name, np.abs(got - want).max())
