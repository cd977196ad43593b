"""Self-play mixtures on the device: ovc_learner_rows against a numpy restatement, ovc_encode_linear_masked against the two-view
K7's rows, ovc_policy_tail_joint against ovc_policy_tail_logp on the same joint rows (with sentinels around what they must not
write and the counter they must advance), and SelfPlayRollout with a network or population partner against self-play and
against AgentPairRollout, bit for bit, over windows whose episodes cross the window boundary."""
import copy

import numpy as np
import pytest
import torch

import policy_reference as P
from helpers import TRACE_FILES, TRACE_IDS, Trace
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import (PARTNER_MEMBER_SALT, PARTNER_SEAT_SALT, AgentPairRollout, BCPolicy, RllibLSTMShapedCNN,
                                         RllibShapedCNN, SelfPlayRollout, _NetworkAgent, member_thresholds)
from rollout_reference import learner_rows_reference, members_reference, seats_reference
from test_gpu_bc_partner import POOL_5X4
from test_gpu_pair_collect import _check_window

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95
SENTINEL = -7


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)




# ------------------------------------------------------------------------------------------------ the kernels


@pytest.mark.parametrize("n", [1, 255, 32771])
@pytest.mark.parametrize("kind", ["self_play", "seat0", "seat1", "mixed"])
def test_learner_rows_matches_the_restatement(n, kind):
    rng = np.random.RandomState(n)
    seat = {"self_play": np.full(n, -1), "seat0": np.zeros(n), "seat1": np.ones(n), "mixed": rng.randint(-1, 2, n)}[kind].astype(np.int32)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    lst, first = (torch.full((n + 32,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(2))
    jrow = torch.full((2 * n + 32,), SENTINEL, dtype=torch.int32, device="cuda")
    rg = torch.full((2 + 32,), SENTINEL, dtype=torch.int32, device="cuda")
    env.learner_rows(_dev(seat, torch.int32), lst[:n], first[:n], jrow[:2 * n], rg[:2])
    wl, wf, wj, count = learner_rows_reference(seat)
    assert np.array_equal(_np(lst[:n]), wl) and np.array_equal(_np(first[:n]), wf)
    assert np.array_equal(_np(jrow[:count]), wj) and _np(rg[:2]).tolist() == [0, count]
    assert (_np(lst[n:]) == SENTINEL).all() and (_np(first[n:]) == SENTINEL).all()
    assert (_np(jrow[count:]) == SENTINEL).all() and (_np(rg[2:]) == SENTINEL).all()


def _masked_case(n, rng, kind):
    """(list entries, first rows, total rows): every environment or none, in a random order, with random masks."""
    if kind == "empty":
        return np.zeros(0, np.int32), np.zeros(0, np.int32), 0
    env = rng.permutation(n) if kind == "permuted" else np.arange(n)
    mask = {"both": np.full(n, 3), "one": rng.randint(1, 3, n), "mixed": rng.randint(0, 4, n), "permuted": rng.randint(0, 4, n)}[kind]
    cnt = np.array([bin(m).count("1") for m in mask])
    return (env << 2 | mask).astype(np.int32), (np.cumsum(cnt) - cnt).astype(np.int32), int(cnt.sum())


@pytest.mark.parametrize("n_layouts", [1, 2, 8])
@pytest.mark.parametrize("n_out", [512, 384, 192], ids=["cpl8", "cpl4", "cpl2"])
def test_encode_linear_masked_equals_the_two_view_rows(n_layouts, n_out):
    n = 700
    rng = np.random.RandomState(n_layouts * 7 + n_out)
    env = BatchedOvercookedEnv(POOL_5X4[:n_layouts], n, horizon=15, env_layout=np.arange(n) % n_layouts, rnd_obj_prob_thresh=0.6,
                               random_start_pos=True, seed=n_layouts)
    env.reset()
    torch.manual_seed(n_out)
    wt = (torch.randn(520, n_out, device="cuda") * 0.2).to(torch.bfloat16)
    bias = torch.randn(n_out, device="cuda") * 0.1
    two = env.encoded_linear(wt, bias)
    for kind in ("empty", "both", "one", "mixed", "permuted"):
        lst, first, total = _masked_case(n, rng, kind)
        out = torch.full((2 * n + 5, n_out), float("nan"), dtype=torch.bfloat16, device="cuda")
        if kind == "empty":  # a list of no entries: a well-formed call of size 0
            l = env.layouts[0]
            ptr = out.data_ptr()
            assert _native.lib().ovc_encode_linear_masked(env.tables.data_ptr(), env.n_layouts, env.state.data_ptr(), ptr, ptr,
                                                          wt.data_ptr(), bias.data_ptr(), ptr, 0, env.state_words, l.width,
                                                          l.height, 15, n_out, 0.2, None) == 0
        else:
            env.encoded_linear_masked(wt, bias, _dev(lst, torch.int32), _dev(first, torch.int32), out)
        want_rows = [2 * (x >> 2) + v for x in lst for v in (0, 1) if x >> v & 1]
        assert len(want_rows) == total
        if total:
            assert torch.equal(out[:total], two[torch.tensor(want_rows, device="cuda")]), kind
        assert torch.isnan(out[total:].float()).all(), kind


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_encode_linear_masked_on_exact_operands_and_every_fixture(path):
    """Certified-exact operands (``policy_reference.k7_operands``) on the fixtures' states: the masked rows equal the float64
    restatement on the oracle's encoding, rounded once to bfloat16."""
    tr = Trace(path)
    st = tr.data["obs_states"]
    n, l = len(st), tr.layout
    if l.width * l.height * 19 * 64 * 2 > 226 * 1024:
        pytest.skip("K7's table of this grid does not fit shared memory")
    env = BatchedOvercookedEnv(l, n, horizon=400)
    env.state.copy_(torch.from_numpy(st))
    rng = np.random.RandomState(l.width * 31 + l.height)
    obs = cpu.encode_lossless(env._tab_host, st, l.width, l.height, env.horizon).astype(np.float64)
    wt, b = P.k7_operands(rng, obs.shape[2] * obs.shape[3] * obs.shape[4], 64)
    want, certs = P.k7_reference(obs.reshape(2 * n, -1), wt, b, 0.2)
    assert certs[0].holds(), "premise: the operands are not exact in float32"
    lst, first, total = _masked_case(n, rng, "permuted")
    out = torch.full((2 * n + 3, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    env.encoded_linear_masked(_dev(wt, torch.bfloat16), _dev(b, torch.float32), _dev(lst, torch.int32), _dev(first, torch.int32), out)
    rows = [2 * (x >> 2) + v for x in lst for v in (0, 1) if x >> v & 1]
    assert np.array_equal(_np(out[:total].float()), want[rows]) and torch.isnan(out[total:].float()).all()


RANGES = [(0, 0), (5, 5), (0, 1), (3, 4), (7, 300), (1, 700), (0, 700), (699, 700), (130, 131), (17, 529)]


def _tail(lib, a, x, n, counter, actions, values, logp, scores, jrow=None, rg=None):
    w1, b1, wh, bh, wo, bo = a._tail
    args = (x.data_ptr(), n, x.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[0], wo.data_ptr(),
            bo.data_ptr(), 0.3, 6, 77, counter.data_ptr())
    if jrow is None:
        _native.check(lib.ovc_policy_tail_logp(*args, actions.data_ptr(), values.data_ptr(), scores.data_ptr(), logp.data_ptr(), 0))
    else:
        _native.check(lib.ovc_policy_tail_joint(*args, jrow.data_ptr(), rg.data_ptr(), actions.data_ptr(), values.data_ptr(),
                                                scores.data_ptr(), logp.data_ptr(), 0))


def test_policy_tail_joint_equals_the_two_view_rows():
    """Compact row r of the joint form equals ovc_policy_tail_logp's joint row jrow[r] (action, value, logp, heads); other
    joint rows and rows outside the range stay untouched; the counter advances by one per launch, also for an empty range,
    and the step crosses 2^32."""
    n = 700  # compact rows; the joint rows are 2 * n
    rng = np.random.RandomState(11)
    torch.manual_seed(11)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    a = _NetworkAgent(env, RllibShapedCNN(5, 4), 0, None, 0, torch.bfloat16)
    lib = _native.lib()
    jrow = np.sort(rng.choice(2 * n, n, replace=False)).astype(np.int32)
    jrow_t = _dev(jrow, torch.int32)
    x = (torch.randn(n, 160, device="cuda") * 2).to(torch.bfloat16)
    x_joint = (torch.randn(2 * n, 160, device="cuda") * 2).to(torch.bfloat16)
    x_joint[jrow_t.long()] = x
    for start in (0, 2**32 - 1):
        for lo, hi in RANGES:
            cj, cr = (torch.tensor([start, 0], dtype=torch.int64, device="cuda") for _ in range(2))
            act_j, act_r = (torch.full((2 * n,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(2))
            val_j, val_r, lp_j, lp_r = (torch.full((2 * n,), float("nan"), device="cuda") for _ in range(4))
            sc_j, sc_r = (torch.full((2 * n, 8), float("nan"), device="cuda") for _ in range(2))
            for _ in range(2):  # two launches: the second draws at step start + 1
                _tail(lib, a, x_joint, 2 * n, cr, act_r, val_r, lp_r, sc_r)
                _tail(lib, a, x, n, cj, act_j, val_j, lp_j, sc_j, jrow_t, torch.tensor([lo, hi], dtype=torch.int32, device="cuda"))
                assert _np(cj).tolist() == _np(cr).tolist()
            assert _np(cj).tolist() == [start + 2, 0]
            listed = np.zeros(2 * n, bool)
            listed[jrow[lo:hi]] = True
            sel, rest = torch.from_numpy(np.nonzero(listed)[0]).cuda(), torch.from_numpy(np.nonzero(~listed)[0]).cuda()
            assert torch.equal(act_j[sel], act_r[sel]) and (act_j[rest] == SENTINEL).all(), (start, lo, hi)
            for got, want in ((val_j, val_r), (lp_j, lp_r), (sc_j, sc_r)):
                assert torch.equal(got[sel], want[sel]) and torch.isnan(got[rest]).all(), (start, lo, hi)


# ------------------------------------------------------------------------------------------------ whole rollouts

FIELDS = ("actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "states", "last_values")


def _selfplay(env, A, seed, graph, **kw):
    return SelfPlayRollout(env, model=copy.deepcopy(A), seed=seed, use_graph=graph, episode_capacity=3, **kw)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_a_network_partner_that_never_plays_changes_nothing(graph):
    """bc_factor = 0: every field of every window, the records and run()'s states equal self-play's."""
    torch.manual_seed(31)
    A, B = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", 517, horizon=13, auto_reset=True)
    sp, mix = _selfplay(mk(), A, 4, graph), _selfplay(mk(), A, 4, graph, partner=B, bc_factor=0.0)
    assert mix._learner_rows
    for w in range(2):
        bs, bm = sp.collect(30, GAMMA, LAM), mix.collect(30, GAMMA, LAM)
        for k in FIELDS:
            assert torch.equal(getattr(bs, k), getattr(bm, k)), (w, k)
        assert (bm.partner_seat == -1).all()
        fs, fm = bs.episodes.finished(), bm.episodes.finished()
        assert len(fs["ep_length"]) > 0
        for k in fs:
            assert torch.equal(fs[k], fm[k]), (w, k)
    sp.run(7), mix.run(7)
    assert torch.equal(sp.env.state, mix.env.state) and torch.equal(sp.actions, mix.actions)


def _seats_follow_the_draw(b, n, seed, bc, shadow, step):
    ps, d = _np(b.partner_seat).astype(np.int32), _np(b.dones)
    for t in range(ps.shape[0]):
        assert np.array_equal(ps[t], shadow), t
        shadow = seats_reference(n, seed ^ PARTNER_SEAT_SALT, step, bc, shadow, d[t])
        step += 1
    return shadow, step


def _masked_equal(bs, bm):
    mask = bm.learner_mask.bool()
    for k in ("actions", "states", "dones"):
        assert torch.equal(getattr(bs, k), getattr(bm, k)), k
    for k in ("logp", "values", "rewards", "advantages"):
        assert torch.equal(getattr(bs, k)[mask], getattr(bm, k)[mask]), k


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_a_copy_of_the_learner_as_partner_draws_what_selfplay_draws(graph):
    """partner = deepcopy(A) at bc_factor 0.5: the actions and states equal self-play's, and so do the learner rows' logp,
    values, rewards and advantages; the seats follow the restated seat draw."""
    n, T, seed = 517, 30, 8
    torch.manual_seed(32)
    A = RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=13, auto_reset=True)
    sp, mix = _selfplay(mk(), A, seed, graph), _selfplay(mk(), A, seed, graph, partner=copy.deepcopy(A), bc_factor=0.5)
    shadow, step = seats_reference(n, seed ^ PARTNER_SEAT_SALT, 0, 0.5, None), 1
    for w in range(2):
        bs, bm = sp.collect(T, GAMMA, LAM), mix.collect(T, GAMMA, LAM)
        _masked_equal(bs, bm)
        shadow, step = _seats_follow_the_draw(bm, n, seed, 0.5, shadow, step)
        assert (bm.partner_seat == -1).any() and (bm.partner_seat >= 0).any()
    sp.run(5), mix.run(5)
    assert torch.equal(sp.env.state, mix.env.state)


def _against_pair(mk, A, partner, seed, graph, lstm=False, T=30, windows=2, **kw):
    """The mixture at bc_factor 1 against AgentPairRollout(A, partner) with random seats: the learner rows of every window
    (with the bootstrap, the LSTM snapshots, the seats and the records), then run()'s joint actions and states."""
    mix = _selfplay(mk(), A, seed, graph, partner=copy.deepcopy(partner), bc_factor=1.0, **kw)
    pair = AgentPairRollout(mk(), (copy.deepcopy(A), copy.deepcopy(partner)), seed=seed, use_graph=graph, random_seats=True,
                            episode_capacity=3, **kw)
    for w in range(windows):
        bm, bp = mix.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        _check_window(bm, bp, pair, lstm, with_seats=True)
        if kw or isinstance(partner, list):
            assert torch.equal(bm.partner_member, bp.partner_member), w
    for _ in range(3):
        mix.run(1), pair.run(1)
        assert torch.equal(mix.actions, pair.actions) and torch.equal(mix.env.state, pair.env.state)
    return mix, pair


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_a_network_partner_at_factor_one_equals_the_pair(lstm, graph):
    torch.manual_seed(33)
    A = RllibLSTMShapedCNN(5, 4) if lstm else RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", 517, horizon=20, auto_reset=True)
    mix, _ = _against_pair(mk, A, RllibShapedCNN(5, 4), 9, graph, lstm=lstm)
    assert mix._learner_rows != lstm  # the LSTM learner keeps the two-view sequence


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_a_population_with_fixed_members_equals_the_pair_population(graph):
    torch.manual_seed(34)
    n = 600
    m = _dev(np.random.RandomState(2).choice(3, n, p=[0.5, 0.3, 0.2]), torch.int32)
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=13, auto_reset=True)
    _against_pair(mk, RllibShapedCNN(5, 4), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), BCPolicy()], 6, graph, member=m)


def test_the_library_path_equals_the_pair_population():
    """The nine 5x4 layouts redrawn at resets: K2 and the library layers for the learner (on all 2N rows) and the members."""
    torch.manual_seed(35)
    n = 400
    m = _dev(np.random.RandomState(3).randint(0, 3, n), torch.int32)
    mk = lambda: BatchedOvercookedEnv(POOL_5X4, n, horizon=9, auto_reset=True, random_layout=True, random_start_pos=True,
                                      rnd_obj_prob_thresh=0.6, seed=5)
    mix, _ = _against_pair(mk, RllibShapedCNN(5, 4), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), BCPolicy()], 4, True, T=12,
                           member=m)
    assert not mix.fused_first_layer and not mix._learner_rows and mix.obs is not None
    mk1 = lambda: BatchedOvercookedEnv(POOL_5X4, n, horizon=9, auto_reset=True, random_layout=True, random_start_pos=True,
                                       rnd_obj_prob_thresh=0.6, seed=6)
    _against_pair(mk1, RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), 5, True, T=12)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_drawn_copies_of_the_learner_equal_selfplay_and_follow_the_draw(graph):
    """[deepcopy(A), deepcopy(A)] drawn per episode at bc_factor 0.5 collects what self-play collects; members change only at
    dones, as the restated draw says (also at the ends of self-play episodes)."""
    n, T, seed = 500, 24, 17
    torch.manual_seed(36)
    A = RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    sp = _selfplay(mk(), A, seed, graph)
    mix = _selfplay(mk(), A, seed, graph, partner=[copy.deepcopy(A), copy.deepcopy(A)], bc_factor=0.5, member_weights=[1.0, 3.0])
    thr = member_thresholds([1.0, 3.0])
    shadow = members_reference(n, seed ^ PARTNER_MEMBER_SALT, 0, thr, None)
    assert np.array_equal(_np(mix.member), shadow)
    step = 1
    for w in range(2):
        bs, bm = sp.collect(T, GAMMA, LAM), mix.collect(T, GAMMA, LAM)
        _masked_equal(bs, bm)
        pm, d = _np(bm.partner_member).astype(np.int32), _np(bm.dones)
        for t in range(T):
            assert np.array_equal(pm[t], shadow), (w, t)
            shadow = members_reference(n, seed ^ PARTNER_MEMBER_SALT, step, thr, shadow, d[t])
            step += 1
        assert set(np.unique(pm).tolist()) == {0, 1}
        fm = bm.episodes.finished()
        assert len(fm["partner_member"]) == int(d.sum())
    sp.run(5), mix.run(5)
    assert torch.equal(sp.env.state, mix.env.state)


def test_factor_member_weights_and_sync_weights_reach_the_captured_graph():
    """A captured mixture and an eager one, changed alike between windows (bc_factor, the draw weights, a member's weights
    refolded), collect the same windows, and each change shows in the batch."""
    n, T = 400, 16
    torch.manual_seed(37)
    A, B, C = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    bc = BCPolicy()
    mixes = [SelfPlayRollout(BatchedOvercookedEnv("cramped_room", n, horizon=8, auto_reset=True), model=copy.deepcopy(A), seed=3,
                             use_graph=g, partner=[copy.deepcopy(B), copy.deepcopy(C), copy.deepcopy(bc)], bc_factor=0.0)
             for g in (True, False)]
    for w in range(4):
        got = [p.collect(T, GAMMA, LAM) for p in mixes]
        for key in ("actions", "logp", "values", "rewards", "dones", "advantages", "partner_member", "partner_seat", "states"):
            assert torch.equal(getattr(got[0], key), getattr(got[1], key)), (w, key)
        if w == 0:
            assert (got[0].partner_seat == -1).all()
        if w >= 2:  # bc_factor 1 since window 1: every episode that started since is paired, and with member 1 only
            late = got[0].partner_seat[T // 2:]
            assert (late >= 0).any() and (got[0].partner_member[T // 2:][late >= 0] == 1).any()
        torch.manual_seed(100 + w)
        delta = [torch.randn_like(q) * 0.05 for q in mixes[0]._pop.agents[1].model.parameters()]
        for p in mixes:
            with torch.no_grad():
                for q, dq in zip(p._pop.agents[1].model.parameters(), delta):
                    q.add_(dq)
            p.sync_weights()
            p.bc_factor = 1.0
            p.member_weights = [0.0, 1.0, 0.0]
    assert mixes[0].member_weights == [0.0, 1.0, 0.0] and mixes[0].bc_factor == 1.0
