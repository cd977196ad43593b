"""A population of partners on the device: ovc_group_members against a stable numpy sort, ovc_assign_members against a numpy
Philox restatement, each rows form against its one-view form on the same environments' rows (with sentinels around what it
must not write and the counter it must advance), and AgentPairRollout with a population against pairs of the learner and
each member, bit for bit."""
import copy

import numpy as np
import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeRecords, EpisodeStats
from overcooked_ai_b200.selfplay import (PARTNER_MEMBER_SALT, AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN,
                                         _NetworkAgent, member_thresholds)
from rollout_reference import members_reference
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95
SENTINEL = -7


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


# ------------------------------------------------------------------------------------------------ grouping


@pytest.mark.parametrize("k,n,kind", [(1, 1000, "random"), (2, 4099, "random"), (7, 32771, "random"), (64, 5000, "random"),
                                      (64, 40, "random"), (7, 3000, "empty_groups"), (5, 2047, "one_group"), (3, 1, "random")])
def test_group_members_is_a_stable_counting_sort(k, n, kind):
    rng = np.random.RandomState(k * 1000 + n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    if kind == "empty_groups":
        m = rng.choice([0, 3, 6], n)
    elif kind == "one_group":
        m = np.full(n, k - 1)
    else:
        m = rng.randint(0, k, n)
    order = torch.full((n + 32,), SENTINEL, dtype=torch.int32, device="cuda")
    offsets = torch.full((k + 1 + 32,), SENTINEL, dtype=torch.int32, device="cuda")
    env.group_members(_dev(m, torch.int32), k, order[:n], offsets[:k + 1])
    want = np.argsort(m, kind="stable")
    counts = np.bincount(m, minlength=k)
    assert np.array_equal(_np(order[:n]), want)
    assert np.array_equal(_np(offsets[:k + 1]), np.concatenate([[0], np.cumsum(counts)]))
    assert (_np(order[n:]) == SENTINEL).all() and (_np(offsets[k + 1:]) == SENTINEL).all()


# ------------------------------------------------------------------------------------------------ the population draw


@pytest.mark.parametrize("n", [1, 255, 4099])
def test_assign_members_matches_the_restatement_and_the_record_slot_rule(n):
    rng = np.random.RandomState(n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    K, seed, cap = 5, 987, 2
    member = torch.zeros(n, dtype=torch.int32, device="cuda")
    thr_dev = torch.zeros(K - 1, dtype=torch.int64, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    rec = EpisodeRecords(env, cap, members=True)
    rec.partner_member.fill_(SENTINEL)
    count = np.zeros(n, np.int64)
    ref = np.zeros(n, np.int32)
    rec_ref = np.full((cap, n), SENTINEL, np.int32)
    weights = ([1, 1, 1, 1, 1], [0, 2, 0, 1, 0], [3, 0, 0, 0, 1], [0, 0, 0, 0, 1], [0.5, 0.25, 1e-3, 0, 2])
    for step, w in enumerate(weights * 2):
        thr = member_thresholds(w)
        thr_dev.copy_(torch.from_numpy(thr))
        done = None if step == 0 else (rng.rand(n) < 0.4).astype(np.int32)
        if done is not None:  # the record slot rule: the member before the draw, into slot count[e] while there is room
            for e in np.nonzero(done)[0]:
                if count[e] < cap:
                    rec_ref[count[e], e] = ref[e]
        env.assign_members(member, K, thr_dev, counter, seed=seed, done=None if done is None else _dev(done, torch.int32), records=rec)
        ref = members_reference(n, seed, step, thr, ref, done)
        got = _np(member)
        assert np.array_equal(got, ref), step
        zero = np.nonzero(np.asarray(w) == 0)[0]
        changed = np.ones(n, bool) if done is None else done != 0
        assert not np.isin(got[changed], zero).any(), step
        assert np.array_equal(_np(rec.partner_member), rec_ref), step
        if done is not None:  # the record kernel's count, advanced here by hand
            count += (done != 0) & (count < cap)
            rec.count.copy_(_dev(count, torch.int32))
    assert _np(counter).tolist() == [len(weights) * 2, 0]
    assert (count == cap).any() or n == 1
    # records only (a fixed member): the counter is left alone and the members stay
    before = member.clone()
    env.assign_members(member, K, done=torch.ones(n, dtype=torch.int32, device="cuda"), records=rec)
    assert torch.equal(member, before) and _np(counter).tolist() == [len(weights) * 2, 0]


def test_member_weights_changed_between_graph_replays_take_effect():
    n, K, seed = 3000, 3, 5
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    member = torch.zeros(n, dtype=torch.int32, device="cuda")
    thr_dev = torch.zeros(K - 1, dtype=torch.int64, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    done = torch.ones(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        env.assign_members(member, K, thr_dev, counter, seed=seed, done=done)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.assign_members(member, K, thr_dev, counter, seed=seed, done=done)
    counter.zero_()
    ref = np.zeros(n, np.int32)
    for step, w in enumerate(([1, 1, 1], [0, 0, 1], [1, 0, 0], [0, 3, 1])):
        thr = member_thresholds(w)
        thr_dev.copy_(torch.from_numpy(thr))
        g.replay()
        ref = members_reference(n, seed, step, thr, ref)
        assert np.array_equal(_np(member), ref), step
    assert set(np.unique(ref).tolist()) == {1, 2}


# ------------------------------------------------------------------------------------------------ the rows forms

RANGES = [(0, 0), (5, 5), (0, 1), (3, 4), (7, 300), (1, 700), (0, 700), (699, 700), (130, 131), (17, 529)]


def _rows_case(n, rng):
    """A random grouping of n environments: (rows int32 [n], seats p(e), swap int32 [n])."""
    return rng.permutation(n).astype(np.int32), rng.randint(0, 2, n)


def _range(lo, hi):
    return torch.tensor([lo, hi], dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("n_layouts", [1, 2, 8])
def test_encode_linear_rows_equals_the_view_rows(n_layouts):
    n = 700
    rng = np.random.RandomState(n_layouts)
    env = BatchedOvercookedEnv(POOL_5X4[:n_layouts], n, horizon=15, env_layout=np.arange(n) % n_layouts, rnd_obj_prob_thresh=0.6,
                               random_start_pos=True, seed=n_layouts)
    env.reset()
    a = _NetworkAgent(env, RllibShapedCNN(5, 4), 0, None, 0, torch.bfloat16)
    rows, swap = _rows_case(n, rng)
    rows_t, swap_t = _dev(rows, torch.int32), _dev(swap, torch.int32)
    for seat in (0, 1):
        view = env.encoded_linear_view(a._wt0, a._b0, seat, swap_t)
        for lo, hi in RANGES:
            out = torch.full_like(view, float("nan"))
            env.encoded_linear_rows(a._wt0, a._b0, seat, swap_t, rows_t, _range(lo, hi), out)
            assert torch.equal(out[lo:hi], view[rows[lo:hi]]), (seat, lo, hi)
            assert torch.isnan(out[:lo]).all() and torch.isnan(out[hi:]).all(), (seat, lo, hi)


def test_wide_layers_range_equals_the_full_call():
    m = 1000
    torch.manual_seed(0)
    env = BatchedOvercookedEnv("cramped_room", m, horizon=400)
    a = _NetworkAgent(env, RllibShapedCNN(5, 4), 0, None, 0, torch.bfloat16)
    w1, b1, w2, b2 = a._wide
    a0 = (torch.randn(m, 512, device="cuda") * 0.5).to(torch.bfloat16)
    lib = _native.lib()
    full = torch.empty(m, 160, dtype=torch.bfloat16, device="cuda")
    _native.check(lib.ovc_wide_layers(a0.data_ptr(), m, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(), 160, 0.2,
                                      full.data_ptr(), 0))
    for lo, hi in RANGES + [(0, 1000), (999, 1000), (1, 999), (300, 2000)]:
        z = torch.full_like(full, float("nan"))
        rg = _range(lo, hi)
        _native.check(lib.ovc_wide_layers_range(a0.data_ptr(), m, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(), 160,
                                                0.2, rg.data_ptr(), z.data_ptr(), 0))
        hi = min(hi, m)
        assert torch.equal(z[lo:hi], full[lo:hi]), (lo, hi)
        assert torch.isnan(z[:lo]).all() and torch.isnan(z[hi:]).all(), (lo, hi)


def _tail_view(lib, a, x, n, counter, swap, seat, actions, values, logp):
    w1, b1, wh, bh, wo, bo = a._tail
    _native.check(lib.ovc_policy_tail_view(x.data_ptr(), n, x.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(),
                                           wh.shape[0], wo.data_ptr(), bo.data_ptr(), 0.3, 6, 77, counter.data_ptr(), swap.data_ptr(), seat,
                                           actions.data_ptr(), values.data_ptr(), 0, 0 if logp is None else logp.data_ptr(), 0))


def _tail_rows(lib, a, x, n, counter, swap, seat, rows, rg, actions, values, logp):
    w1, b1, wh, bh, wo, bo = a._tail
    _native.check(lib.ovc_policy_tail_rows(x.data_ptr(), n, x.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(),
                                           wh.shape[0], wo.data_ptr(), bo.data_ptr(), 0.3, 6, 77, counter.data_ptr(), swap.data_ptr(), seat,
                                           rows.data_ptr(), rg.data_ptr(), actions.data_ptr(), values.data_ptr(), 0,
                                           0 if logp is None else logp.data_ptr(), 0))


@pytest.mark.parametrize("with_logp", [False, True], ids=["plain", "logp"])
@pytest.mark.parametrize("kernel", ["policy_tail", "sample_actions"])
def test_rows_draws_equal_the_view_draws(kernel, with_logp):
    """Compact row r of the rows form equals the one-view form's row rows[r]: the action at its joint row, its value and logp;
    the other seat, other environments' entries and rows outside the range stay untouched; the counter advances by one per
    launch, also for an empty range, and the step crosses 2^32."""
    n = 700
    rng = np.random.RandomState(11)
    torch.manual_seed(11)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    a = _NetworkAgent(env, RllibShapedCNN(5, 4), 0, None, 0, torch.bfloat16)
    lib = _native.lib()
    rows, swap = _rows_case(n, rng)
    rows_t, swap_t = _dev(rows, torch.int32), _dev(swap, torch.int32)
    x = (torch.randn(n, 160, device="cuda") * 2).to(torch.bfloat16)  # compact rows: row r belongs to environment rows[r]
    scores = torch.randn(n, 8, device="cuda") * 3
    x_env, scores_env = torch.empty_like(x), torch.empty_like(scores)  # the same rows by environment, for the view forms
    x_env[rows_t.long()], scores_env[rows_t.long()] = x, scores
    for start in (0, 2**32 - 1):
        for seat in (0, 1):
            p = seat ^ swap
            for lo, hi in RANGES:
                cv, cr = (torch.tensor([start, 0], dtype=torch.int64, device="cuda") for _ in range(2))
                act_v = torch.full((n, 2), SENTINEL, dtype=torch.int32, device="cuda")
                act_r = torch.full((n, 2), SENTINEL, dtype=torch.int32, device="cuda")
                val_v, val_r, lp_v, lp_r = (torch.full((n,), float("nan"), device="cuda") for _ in range(4))
                for _ in range(2):  # two launches: the second draws at step start + 1
                    if kernel == "policy_tail":
                        _tail_view(lib, a, x_env, n, cv, swap_t, seat, act_v, val_v, lp_v if with_logp else None)
                        _tail_rows(lib, a, x, n, cr, swap_t, seat, rows_t, _range(lo, hi), act_r, val_r, lp_r if with_logp else None)
                    else:
                        env.sample_actions_view(scores_env, cv, seat, swap_t, seed=77, out=act_v, logp_out=lp_v if with_logp else None)
                        env.sample_actions_rows(scores, cr, seat, swap_t, rows_t, _range(lo, hi), seed=77, out=act_r,
                                                logp_out=lp_r if with_logp else None)
                    assert _np(cr).tolist() == _np(cv).tolist()
                assert _np(cr).tolist() == [start + 2, 0]
                av, ar = _np(act_v), _np(act_r)
                want = np.full((n, 2), SENTINEL, np.int32)
                e = rows[lo:hi]
                want[e, p[e]] = av[e, p[e]]
                assert np.array_equal(ar, want), (start, seat, lo, hi)
                et = rows_t[lo:hi].long()
                if kernel == "policy_tail":
                    assert torch.equal(val_r[lo:hi], val_v[et]) and torch.isnan(val_r[:lo]).all() and torch.isnan(val_r[hi:]).all()
                if with_logp:
                    assert torch.equal(lp_r[lo:hi], lp_v[et]) and torch.isnan(lp_r[:lo]).all() and torch.isnan(lp_r[hi:]).all()


# ------------------------------------------------------------------------------------------------ whole rollouts


def _select(n, m, k):
    return torch.from_numpy(np.nonzero(m == k)[0]).cuda()


def _fixed_members(make_env, A, members, m, seed, graph, T=20, windows=2):
    """A population with a fixed member tensor m against one pair (A, member k) per member: on the environments with m == k
    the collect() batches, the episode records, run()'s states and records equal the pair's bit for bit."""
    K = len(members)
    pop = AgentPairRollout(make_env(), (copy.deepcopy(A), [copy.deepcopy(x) for x in members]), seed=seed, random_seats=True,
                           member=_dev(m, torch.int32), use_graph=graph, episode_capacity=3)
    pairs = [AgentPairRollout(make_env(), (copy.deepcopy(A), copy.deepcopy(x)), seed=seed, random_seats=True, use_graph=graph,
                              episode_capacity=3) for x in members]
    for w in range(windows):
        bp = pop.collect(T, GAMMA, LAM)
        bks = [q.collect(T, GAMMA, LAM) for q in pairs]
        fp = bp.episodes.finished()
        assert len(fp["env_index"]) > 0
        for k in range(K):
            sel, bk = _select(pop.env.n_envs, m, k), bks[k]
            for key in ("actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "partner_seat", "states"):
                assert torch.equal(getattr(bp, key)[:, sel], getattr(bk, key)[:, sel]), (w, k, key)
            assert torch.equal(bp.last_values[sel], bk.last_values[sel]) and (bp.partner_member[:, sel] == k).all()
            fk = bk.episodes.finished()
            ip, ik = torch.isin(fp["env_index"], sel), torch.isin(fk["env_index"], sel)
            for key in fk:
                assert torch.equal(fp[key][ip], fk[key][ik]), (w, k, key)
            assert (fp["partner_member"][ip] == k).all()
            assert torch.equal(pop.env.state[sel], pairs[k].env.state[sel]), (w, k)
    for q in [pop] + pairs:
        q.run(T)
    fp = pop.episodes.finished()
    for k in range(K):
        sel = _select(pop.env.n_envs, m, k)
        assert torch.equal(pop.env.state[sel], pairs[k].env.state[sel]), k
        fk = pairs[k].episodes.finished()
        ip, ik = torch.isin(fp["env_index"], sel), torch.isin(fk["env_index"], sel)
        for key in fk:
            assert torch.equal(fp[key][ip], fk[key][ik]), (k, key)
        assert (fp["partner_member"][ip] == k).all()
    return pop


@pytest.mark.parametrize("lstm", [False, True], ids=["cnn", "lstm"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_fixed_members_equal_their_pairs(lstm, graph):
    torch.manual_seed(21)
    A = RllibLSTMShapedCNN(5, 4) if lstm else RllibShapedCNN(5, 4)
    members = [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), BCPolicy()]
    n = 600
    m = np.random.RandomState(2).choice(3, n, p=[0.5, 0.3, 0.2]).astype(np.int32)
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=13, auto_reset=True)
    pop = _fixed_members(mk, A, members, m, 6, graph)
    assert all(a.fused_first_layer and a.fused_wide and a.fused_tail for a in pop.agents[1].agents[:2])


def test_fixed_members_on_the_library_path_equal_their_pairs():
    """The nine 5x4 layouts redrawn at resets: more than K7 takes, so K2 -> the library layers on all compact rows -> K8's rows
    form for each member."""
    torch.manual_seed(22)
    n = 400
    m = np.random.RandomState(3).randint(0, 3, n).astype(np.int32)
    mk = lambda: BatchedOvercookedEnv(POOL_5X4, n, horizon=9, auto_reset=True, random_layout=True, random_start_pos=True,
                                      rnd_obj_prob_thresh=0.6, seed=5)
    pop = _fixed_members(mk, RllibShapedCNN(5, 4), [RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), BCPolicy()], m, 4, True, T=12)
    assert pop.obs is not None and not pop.agents[1].agents[0].fused_first_layer and pop.agents[1].agents[0].fused_tail


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_drawn_copies_of_one_member_equal_the_pair_and_follow_the_draw(graph):
    """(A, [B, deepcopy(B)]) draws what (A, B) draws whatever member is drawn; members change only at dones, as the restated
    draw says, and every finished episode's member is the one of its last step."""
    n, T, seed = 500, 24, 17
    torch.manual_seed(23)
    A, B = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    mk = lambda: BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    pop = AgentPairRollout(mk(), (copy.deepcopy(A), [copy.deepcopy(B), copy.deepcopy(B)]), seed=seed, random_seats=True,
                           member_weights=[1.0, 3.0], use_graph=graph, episode_capacity=4)
    pair = AgentPairRollout(mk(), (copy.deepcopy(A), copy.deepcopy(B)), seed=seed, random_seats=True, use_graph=graph, episode_capacity=4)
    thr = member_thresholds([1.0, 3.0])
    shadow = members_reference(n, seed ^ PARTNER_MEMBER_SALT, 0, thr, None)
    assert np.array_equal(_np(pop.member), shadow)
    step = 1
    for w in range(2):
        bp, bq = pop.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        for key in ("actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "partner_seat", "states", "last_values"):
            assert torch.equal(getattr(bp, key), getattr(bq, key)), (w, key)
        pm, d = _np(bp.partner_member).astype(np.int32), _np(bp.dones)
        for t in range(T):
            assert np.array_equal(pm[t], shadow), (w, t)
            shadow = members_reference(n, seed ^ PARTNER_MEMBER_SALT, step, thr, shadow, d[t])
            step += 1
        assert np.array_equal(_np(pop.member), shadow)
        fp, fq = bp.episodes.finished(), bq.episodes.finished()
        for key in fq:
            assert torch.equal(fp[key], fq[key]), (w, key)
        # the episode that ended at transition t was played with member pm[t] (slot order: per environment, by time)
        ends = [(e, t) for e in range(n) for t in range(T) if d[t, e]]
        got = {}
        for e, mem in zip(_np(fp["env_index"]).tolist(), _np(fp["partner_member"]).tolist()):
            got.setdefault(e, []).append(mem)
        want = {}
        for e, t in ends:
            want.setdefault(e, []).append(int(pm[t, e]))
        assert got == want
        assert set(np.unique(pm).tolist()) == {0, 1}
    pop.run(5), pair.run(5)
    assert torch.equal(pop.env.state, pair.env.state)


def test_sync_weights_and_member_weights_reach_the_captured_graph():
    """A captured population and an eager one, changed alike between windows (a member's weights refolded, the draw weights
    moved to a single member), collect the same windows."""
    n, T = 400, 16
    torch.manual_seed(24)
    A, B, C = RllibShapedCNN(5, 4), RllibShapedCNN(5, 4), RllibShapedCNN(5, 4)
    pops = [AgentPairRollout(BatchedOvercookedEnv("cramped_room", n, horizon=8, auto_reset=True),
                             (copy.deepcopy(A), [copy.deepcopy(B), copy.deepcopy(C), BCPolicy()]), seed=3, random_seats=True,
                             use_graph=g) for g in (True, False)]
    for p in pops[1:]:  # the same BC member in both
        p.agents[1].agents[2].policy.load_state_dict(pops[0].agents[1].agents[2].policy.state_dict())
        p.agents[1].agents[2].sync_weights()
    for w in range(3):
        got = [p.collect(T, GAMMA, LAM) for p in pops]
        for key in ("actions", "logp", "values", "rewards", "dones", "advantages", "partner_member", "states"):
            assert torch.equal(getattr(got[0], key), getattr(got[1], key)), (w, key)
        torch.manual_seed(100 + w)
        delta = [torch.randn_like(q) * 0.05 for q in pops[0].agents[1].agents[1].model.parameters()]
        for p in pops:
            with torch.no_grad():
                for q, dq in zip(p.agents[1].agents[1].model.parameters(), delta):
                    q.add_(dq)
            p.sync_weights()
            p.member_weights = [0.0, 1.0, 0.0] if w == 0 else [1.0, 1.0, 2.0]
    assert pops[0].member_weights == [1.0, 1.0, 2.0]
    b = pops[0].collect(T, GAMMA, LAM)  # after [0, 1, 0]: every episode that started since plays member 1
    assert bool((b.partner_member == 1).any())
