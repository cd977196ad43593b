"""Population play on the device: ovc_assign_pairs against a numpy Philox restatement, ovc_group_pairs against a numpy
restatement of its layout, ovc_encode_linear_grouped_masked against ovc_encode_linear per member, ovc_policy_tail_grouped_joint
against ovc_policy_tail_logp per member at the joint rows (sentinels past the end, the counter advanced once), and
SelfPlayRollout with pairs / pair_weights: copies of one model equal self-play bit for bit, diagonal pairs equal blocks,
distinct members equal each member's own policy on its rows, the pairing invariants and sync_weights."""
import copy

import numpy as np
import pytest
import torch

import limit_layouts as LL
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeRecords
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout, pair_thresholds, PAIR_SALT
from rollout_reference import pairs_reference
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95
SENTINEL = -7


def _np(t):
    return t.cpu().numpy()


def _dev(a, dt=torch.int32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()


# ------------------------------------------------------------------------------------------------ ovc_assign_pairs


@pytest.mark.parametrize("K,n", [(1, 33), (3, 255), (8, 4099), (64, 1000)])
def test_assign_pairs_matches_the_restatement_and_the_record_slot_rule(K, n):
    rng = np.random.RandomState(K * 7 + n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    seed, cap = 0xABCDEF ^ K, 2
    rec = EpisodeRecords(env, cap, pairs=True)
    pair = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    ref = np.zeros((n, 2), np.int32)
    rec_ref = np.zeros((cap, n, 2), np.int32)
    count = np.zeros(n, np.int32)
    thr_dev = torch.zeros(max(K * K - 1, 1), dtype=torch.int64, device="cuda")
    for step in range(6):
        w = rng.rand(K, K) * (rng.rand(K, K) < 0.5)
        w[rng.randint(K), rng.randint(K)] += 1.0
        thr = pair_thresholds(w, K)
        thr_dev[:K * K - 1].copy_(torch.from_numpy(thr))
        done = None if step == 0 else (rng.rand(n) < 0.4).astype(np.int32)
        if done is not None:
            for e in np.nonzero(done)[0]:
                if count[e] < cap:
                    rec_ref[count[e], e] = ref[e]
        env.assign_pairs(pair, K, thr_dev, counter, seed=seed, done=None if done is None else _dev(done), records=None if done is None else rec)
        ref = pairs_reference(n, K, seed, step, thr, ref, done)
        got = _np(pair)
        assert np.array_equal(got, ref), step
        changed = np.flatnonzero(done != 0) if done is not None else np.arange(n)
        assert (w[got[changed, 0], got[changed, 1]] > 0).all(), "a pair of weight 0 is never drawn"
        if done is not None:  # the record transition would bump count after the record: do it by hand
            count = np.minimum(count + (done != 0), cap)
            rec.count.copy_(_dev(count))
        assert _np(counter).tolist() == [step + 1, 0], "the step advances exactly once per launch"
    assert np.array_equal(_np(rec.pair), rec_ref)
    assert (count == cap).any()
    # a full buffer writes nothing; records only (fixed pairs): the counter and the pairs stay
    before_rec, before = rec.pair.clone(), pair.clone()
    full = torch.full((n,), cap, dtype=torch.int32, device="cuda")
    rec.count.copy_(full)
    env.assign_pairs(pair, K, done=torch.ones(n, dtype=torch.int32, device="cuda"), records=rec)
    assert torch.equal(rec.pair, before_rec) and torch.equal(pair, before) and _np(counter).tolist() == [6, 0]


# ------------------------------------------------------------------------------------------------ ovc_group_pairs


def group_pairs_reference(pair, K):
    """numpy restatement of ovc_group_pairs: (list, first, jrow, entry_offsets, row_offsets), list / first over the entries."""
    groups = [[] for _ in range(K)]
    for e, (i, j) in enumerate(pair):
        if i == j:
            groups[i].append(e << 2 | 3)
        else:
            groups[i].append(e << 2 | 1)
            groups[j].append(e << 2 | 2)
    lst, first, jrow, eo, ro = [], [], [], [0], [0]
    for g in groups:
        for entry in g:
            e, m = entry >> 2, entry & 3
            lst.append(entry)
            first.append(len(jrow))
            jrow += [2 * e + v for v in (0, 1) if m >> v & 1]
        eo.append(len(lst))
        ro.append(len(jrow))
    return [np.array(a, np.int32) for a in (lst, first, jrow, eo, ro)]


def _pairings(K, n, rng):
    out = {"diagonal": np.repeat(rng.randint(K, size=(n, 1)), 2, 1), "cross": rng.randint(K, size=(n, 2))}
    if K > 1:
        c = out["cross"]
        c[c[:, 0] == c[:, 1], 1] = (c[c[:, 0] == c[:, 1], 0] + 1) % K  # every pair a cross pair
        out["empty_members"] = rng.choice([0, K - 1], size=(n, 2))  # members 1 .. K - 2 have no entry
    return out


@pytest.mark.parametrize("n", [1, 1000, 4099])
@pytest.mark.parametrize("K", [1, 3, 64])
def test_group_pairs_matches_the_restatement(K, n):
    rng = np.random.RandomState(K * 31 + n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    pad = 5
    for name, pr in _pairings(K, n, rng).items():
        bufs = [torch.full((2 * n + pad,), SENTINEL, dtype=torch.int32, device="cuda") for _ in range(3)]
        eo = torch.full((K + 1,), SENTINEL, dtype=torch.int32, device="cuda")
        ro = torch.full((K + 1,), SENTINEL, dtype=torch.int32, device="cuda")
        env.group_pairs(_dev(pr), K, *[b[:2 * n] for b in bufs], eo, ro)
        lst, first, jrow, eo_r, ro_r = group_pairs_reference(pr, K)
        m = len(lst)
        assert np.array_equal(_np(eo), eo_r) and np.array_equal(_np(ro), ro_r), name
        assert ro_r[-1] == 2 * n
        assert np.array_equal(_np(bufs[0])[:m], lst) and np.array_equal(_np(bufs[1])[:m], first), name
        assert np.array_equal(_np(bufs[2])[:2 * n], jrow), name
        for b in bufs:
            assert (_np(b)[2 * n:] == SENTINEL).all(), name


# ------------------------------------------------------------------------------------------------ grouped masked K7


def _grouped_masked(env, wt, bias, pr, K, n_out):
    n = env.n_envs
    lst, first, jrow = (torch.empty(2 * n, dtype=torch.int32, device="cuda") for _ in range(3))
    eo, ro = (torch.empty(K + 1, dtype=torch.int32, device="cuda") for _ in range(2))
    env.group_pairs(pr, K, lst, first, jrow, eo, ro)
    out = torch.full((2 * n + 5, n_out), float("nan"), dtype=torch.bfloat16, device="cuda")
    W, H = env.layouts[0].width, env.layouts[0].height
    _native.check(_native.lib().ovc_encode_linear_grouped_masked(
        env.tables.data_ptr(), env.n_layouts, env.state.data_ptr(), lst.data_ptr(), first.data_ptr(), wt.data_ptr(), bias.data_ptr(),
        eo.data_ptr(), K, out.data_ptr(), 2 * n, env.state_words, W, H, env.horizon, n_out, 0.2, None))
    return out, jrow, ro


def _check_grouped_masked(env, K, n_out, seed):
    rng = np.random.RandomState(seed)
    n = env.n_envs
    W, H = env.layouts[0].width, env.layouts[0].height
    wt = (torch.randn(K, W * H * 26, n_out, device="cuda") * 0.2).to(torch.bfloat16)
    bias = torch.randn(K, n_out, device="cuda") * 0.1
    for name, pr in _pairings(K, n, rng).items():
        out, jrow, ro = _grouped_masked(env, wt, bias, _dev(pr), K, n_out)
        jr, roh = _np(jrow).astype(np.int64), _np(ro)
        for k in range(K):
            a, b = int(roh[k]), int(roh[k + 1])
            if a == b:
                continue
            want = env.encoded_linear(wt[k].contiguous(), bias[k].contiguous())
            assert torch.equal(out[a:b], want[torch.from_numpy(jr[a:b]).cuda()]), (name, k)
        assert torch.isnan(out[2 * n:].float()).all(), name


@pytest.mark.parametrize("K", [1, 3, 64])
def test_grouped_masked_encode_equals_the_encoding_of_each_member(K):
    env = BatchedOvercookedEnv(POOL_5X4[:8], 1031, horizon=15, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=K,
                               env_layout=np.arange(1031) % 8)
    env.reset()
    _check_grouped_masked(env, K, 512, K + 5)


def test_grouped_masked_encode_on_the_largest_k7_grid():
    env = BatchedOvercookedEnv(LL.k7_layouts(13, 7), 8 * 37 + 3, horizon=60, auto_reset=True, random_start_pos=True,
                               rnd_obj_prob_thresh=0.6, seed=3)
    env.reset()
    _check_grouped_masked(env, 3, 128, 9)


# ------------------------------------------------------------------------------------------------ grouped joint K8


def _tables(rng, K, k0, n_hidden):
    bf = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda().to(torch.bfloat16)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    nh = max(n_hidden, 1)
    return (bf(rng.normal(size=(K, 64, k0)) / np.sqrt(k0)), f32(rng.normal(size=(K, 64)) * 0.1),
            bf(rng.normal(size=(K, nh, 64, 64)) / 8), f32(rng.normal(size=(K, nh, 64)) * 0.1),
            bf(rng.normal(size=(K, 8, 64)) / 4), f32(rng.normal(size=(K, 8)) * 0.1))


@pytest.mark.parametrize("k0,n_hidden", [(160, 2), (64, 0), (256, 3)])
@pytest.mark.parametrize("K", [1, 3, 64])
def test_grouped_joint_tail_equals_the_tail_of_each_member_at_the_joint_rows(K, k0, n_hidden):
    lib = _native.lib()
    rng = np.random.RandomState(K * 1000 + k0 + n_hidden)
    n = 2053
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    pr = _pairings(K, n, rng)["cross" if K > 1 else "diagonal"]
    pr[: n // 3] = np.repeat(pr[: n // 3, :1], 2, 1)  # a third self-play pairs
    lst, first, jrow = (torch.empty(2 * n, dtype=torch.int32, device="cuda") for _ in range(3))
    eo, ro = (torch.empty(K + 1, dtype=torch.int32, device="cuda") for _ in range(2))
    env.group_pairs(_dev(pr), K, lst, first, jrow, eo, ro)
    rows, pad = 2 * n, 37
    x = torch.from_numpy(rng.normal(size=(rows, k0)).astype(np.float32)).cuda().to(torch.bfloat16)
    w1, b1, wh, bh, wo, bo = _tables(rng, K, k0, n_hidden)
    seed = 0x1234_5678_9ABC_DEF0 + K
    counter = torch.tensor([41, 0], dtype=torch.int64, device="cuda")
    acts = torch.full((rows + pad,), SENTINEL, dtype=torch.int32, device="cuda")
    vals, lp = (torch.full((rows + pad,), float(SENTINEL), device="cuda") for _ in range(2))
    scores = torch.full((rows + pad, 8), float(SENTINEL), device="cuda")
    _native.check(lib.ovc_policy_tail_grouped_joint(
        x.data_ptr(), rows, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), n_hidden, wo.data_ptr(), bo.data_ptr(),
        0.3, 6, seed, counter.data_ptr(), jrow.data_ptr(), ro.data_ptr(), K, acts.data_ptr(), vals.data_ptr(), scores.data_ptr(),
        lp.data_ptr(), None))
    assert _np(counter).tolist() == [42, 0], "the step advances exactly once per launch"
    jr, roh = _np(jrow).astype(np.int64), _np(ro)
    assert sorted(jr.tolist()) == list(range(rows))
    for k in range(K):
        a, b = int(roh[k]), int(roh[k + 1])
        if a == b:
            continue
        # member k's tables on the x rows scattered to their joint rows: ovc_policy_tail_logp at joint row jrow[r]
        xj = torch.zeros_like(x)
        idx = torch.from_numpy(jr[a:b]).cuda()
        xj[idx] = x[a:b]
        c = torch.tensor([41, 0], dtype=torch.int64, device="cuda")
        ra = torch.empty(rows, dtype=torch.int32, device="cuda")
        rv, rl = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
        rs = torch.empty((rows, 8), device="cuda")
        _native.check(lib.ovc_policy_tail_logp(
            xj.data_ptr(), rows, k0, 0.2, w1[k].data_ptr(), b1[k].data_ptr(), wh[k].data_ptr(), bh[k].data_ptr(), n_hidden, wo[k].data_ptr(),
            bo[k].data_ptr(), 0.3, 6, seed, c.data_ptr(), ra.data_ptr(), rv.data_ptr(), rs.data_ptr(), rl.data_ptr(), None))
        for got, want in ((acts, ra), (vals, rv), (lp, rl), (scores, rs)):
            assert torch.equal(got[idx], want[idx]), k
    for t in (acts, vals, lp, scores):
        assert (_np(t[rows:]) == SENTINEL).all()
    assert len(np.unique(_np(acts[:rows]))) == 6


def test_grouped_joint_tail_leaves_rows_outside_every_member_alone():
    lib = _native.lib()
    rng = np.random.RandomState(5)
    K, k0, rows = 3, 160, 600
    jrow = _dev(rng.permutation(rows))
    ro = _dev(np.array([10, 10, 300, 550]))  # compact rows [0, 10) and [550, 600) belong to no member; member 0 is empty
    x = torch.from_numpy(rng.normal(size=(rows, k0)).astype(np.float32)).cuda().to(torch.bfloat16)
    w1, b1, wh, bh, wo, bo = _tables(rng, K, k0, 2)
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    acts = torch.full((rows,), SENTINEL, dtype=torch.int32, device="cuda")
    vals, lp = (torch.full((rows,), float(SENTINEL), device="cuda") for _ in range(2))
    _native.check(lib.ovc_policy_tail_grouped_joint(
        x.data_ptr(), rows, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), 2, wo.data_ptr(), bo.data_ptr(), 0.3, 6, 9,
        counter.data_ptr(), jrow.data_ptr(), ro.data_ptr(), K, acts.data_ptr(), vals.data_ptr(), 0, lp.data_ptr(), None))
    assert _np(counter).tolist() == [1, 0]
    untouched = _np(jrow)[np.r_[0:10, 550:600]]
    touched = _np(jrow)[10:550]
    assert (_np(acts)[untouched] == SENTINEL).all() and (_np(vals)[untouched] == SENTINEL).all() and (_np(lp)[untouched] == SENTINEL).all()
    assert (_np(acts)[touched] != SENTINEL).all()


# ------------------------------------------------------------------------------------------------ the rollout


def _models(K, W=5, H=4, seed=0):
    out = []
    for k in range(K):
        torch.manual_seed(seed * 100 + k)
        out.append(RllibShapedCNN(W, H))
    return out


CASES = {  # (environment factory for n envs, grid, fused flags (K7, K9, K8))
    "cramped_room": (lambda n: BatchedOvercookedEnv("cramped_room", n, horizon=11, auto_reset=True), (5, 4), (True, True, True)),
    "random_starts": (lambda n: BatchedOvercookedEnv("cramped_room", n, horizon=13, auto_reset=True, random_start_pos=True,
                                                     rnd_obj_prob_thresh=0.5, seed=3), (5, 4), (True, True, True)),
    "grid_5x5": (lambda n: BatchedOvercookedEnv("coordination_ring", n, horizon=12, auto_reset=True), (5, 5), (True, False, False)),
    "pool_8": (lambda n: BatchedOvercookedEnv(POOL_5X4[:8], n, horizon=10, auto_reset=True, env_layout=np.arange(n) % 8),
               (5, 4), (True, True, True)),
}
BATCH_FIELDS = ("states", "actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "last_values")


def _equal_batches(bp, bs):
    for f in BATCH_FIELDS:
        assert torch.equal(getattr(bp, f), getattr(bs, f)), f
    fp, fs = bp.episodes.finished(), bs.episodes.finished()
    assert len(fs["env_index"]) > 0, "premise: episodes end in the window"
    for f in fs:
        assert torch.equal(fp[f], fs[f]), f


def _equal_live(pop, single):
    assert torch.equal(pop.env.state, single.env.state) and torch.equal(pop.actions, single.actions)
    assert torch.equal(pop.values, single.values) and torch.equal(pop.ret_mixed, single.ret_mixed)
    assert torch.equal(pop.ret_sparse, single.ret_sparse)
    fp, fs = pop.episodes.finished(), single.episodes.finished()
    assert len(fs["env_index"]) > 0
    for f in fs:
        assert torch.equal(fp[f], fs[f]), f


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case,K", [("cramped_room", 2), ("cramped_room", 4), ("random_starts", 4), ("grid_5x5", 3), ("pool_8", 2)])
def test_copies_with_uniform_pair_weights_equal_selfplay(case, K, graph):
    make, (W, H), flags = CASES[case]
    model = _models(1, W, H, seed=len(case))[0]
    kw = dict(seed=77, use_graph=graph, episode_capacity=4)
    pop = SelfPlayRollout(make(300), [copy.deepcopy(model) for _ in range(K)], pair_weights=np.ones((K, K)), **kw)
    single = SelfPlayRollout(make(300), model, **kw)
    assert (pop.fused_first_layer, pop.fused_wide, pop.fused_tail) == flags
    first = pop.pair.clone()
    for w in range(2):  # two windows: episodes cross the boundary
        bp, bs = pop.collect(25, GAMMA, LAM), single.collect(25, GAMMA, LAM)
        _equal_batches(bp, bs)
    assert not torch.equal(first, pop.pair), "premise: the pairs were redrawn"
    assert len(np.unique(_np(bp.pair).reshape(-1, 2), axis=0)) == K * K, "premise: every ordered pair played"
    for s in (pop, single):
        s.episodes.clear()
    pop.run(30), single.run(30)
    _equal_live(pop, single)


def test_copies_with_use_phi_equal_selfplay():
    make = CASES["cramped_room"][0]
    model = _models(1, seed=4)[0]
    pop = SelfPlayRollout(make(301), [copy.deepcopy(model) for _ in range(4)], pair_weights=np.ones((4, 4)), seed=5, use_phi=True,
                          episode_capacity=4)
    single = SelfPlayRollout(make(301), model, seed=5, use_phi=True, episode_capacity=4)
    for w in range(2):
        _equal_batches(pop.collect(24, GAMMA, LAM), single.collect(24, GAMMA, LAM))


@pytest.mark.parametrize("K", [2, 4])
def test_diagonal_pairs_equal_blocks(K):
    make = CASES["random_starts"][0]
    blocks = [1, 7, 129, 163] if K == 4 else [137, 163]
    n = sum(blocks)
    models = _models(K, seed=9)
    member = np.repeat(np.arange(K), blocks)
    pairs = _dev(np.stack([member, member], 1))
    kw = dict(seed=123, episode_capacity=4)
    pp = SelfPlayRollout(make(n), models, pairs=pairs, **kw)
    pb = SelfPlayRollout(make(n), models, blocks=blocks, **kw)
    for w in range(2):
        _equal_batches(pp.collect(25, GAMMA, LAM), pb.collect(25, GAMMA, LAM))
    pp.episodes.clear(), pb.episodes.clear()
    pp.run(20), pb.run(20)
    _equal_live(pp, pb)
    assert torch.equal(pp.pair, pairs), "fixed pairs never change"


def _own_policy(pop, f, env, states, counter_step):
    """Member f's two-view K7 -> K9 -> K8 on the records ``states`` [N, S] at the given counter step: (logits [2N, 8],
    values, logp, actions)."""
    lib, N = _native.lib(), env.n_envs
    saved = env.state.clone()
    env.state.copy_(states)
    act0 = env.encoded_linear(f._wt0, f._b0, neg_slope=0.2)
    z = torch.empty((2 * N, f._tail[0].shape[1]), dtype=torch.bfloat16, device="cuda")
    _native.check(lib.ovc_wide_layers(*f._k9_args(act0), z.data_ptr(), None))
    counter = torch.tensor([counter_step, 0], dtype=torch.int64, device="cuda")
    acts = torch.empty(2 * N, dtype=torch.int32, device="cuda")
    vals, lp = torch.empty(2 * N, device="cuda"), torch.empty(2 * N, device="cuda")
    scores = torch.empty((2 * N, 8), device="cuda")
    _native.check(lib.ovc_policy_tail_logp(*pop._k8_args(z, f._tail), counter.data_ptr(), acts.data_ptr(), vals.data_ptr(), scores.data_ptr(), lp.data_ptr(), None))
    env.state.copy_(saved)
    return scores, vals, lp, acts


@pytest.mark.parametrize("K", [2, 3, 4, 5])  # K9 per member at 2 and 3, grouped from 4 on
def test_distinct_members_act_as_their_own_policy_on_their_rows(K):
    make = CASES["random_starts"][0]
    pop = SelfPlayRollout(make(400), _models(K, seed=K), pair_weights=np.ones((K, K)), seed=31, episode_capacity=4)
    T = 20
    b = pop.collect(T, GAMMA, LAM, keep_logits=True)
    N = pop.env.n_envs
    rows_member = b.pair.view(T, 2 * N).long()
    for t in range(0, T, 3):
        for k, f in enumerate([pop] + pop._learners.others):
            mine = rows_member[t] == k
            if not mine.any():
                continue
            scores, vals, lp, acts = _own_policy(pop, f, pop.env, b.states[t], t)
            assert torch.equal(b.logits[t][mine], scores[mine]), (t, k)
            assert torch.equal(b.values[t][mine], vals[mine]) and torch.equal(b.logp[t][mine], lp[mine]), (t, k)
            assert torch.equal(b.actions[t][mine], acts[mine]), (t, k)


def test_pairing_invariants_and_the_weights_setter():
    make = CASES["cramped_room"][0]
    K, N, T = 3, 2000, 33
    pop = SelfPlayRollout(make(N), _models(K, seed=2), pair_weights=np.ones((K, K)), seed=8, episode_capacity=4)
    b = pop.collect(T, GAMMA, LAM)
    pr, dones = _np(b.pair).astype(np.int32), _np(b.dones).astype(bool)
    assert np.array_equal(pr[1:][~dones[:-1]], pr[:-1][~dones[:-1]]), "a pair changes only at a done"
    assert (pr[1:][dones[:-1]] != pr[:-1][dones[:-1]]).any()
    # finished()["pair"] is the pair of the episode's last transition
    fin = b.episodes.finished()
    t_end = {e: list(np.flatnonzero(dones[:, e])) for e in range(N)}
    want = []
    for k_, e in zip(*np.nonzero(np.arange(b.episodes.capacity)[:, None] < _np(b.episodes.count)[None, :])):
        want.append(pr[t_end[e][k_], e])
    assert np.array_equal(_np(fin["pair"]), np.array(want))
    # a new weight matrix through the setter (the captured graph is kept): only (2, 0) from the next dones on
    g = pop._collect_graphs[(T, False)][1]
    w = np.zeros((K, K))
    w[2, 0] = 1.0
    pop.pair_weights = w
    b = pop.collect(T, GAMMA, LAM)
    assert pop._collect_graphs[(T, False)][1] is g
    pr, dones = _np(b.pair).astype(np.int32), _np(b.dones).astype(bool)
    after = np.cumsum(dones, 0) > 0  # transitions after an episode end in this window
    assert (pr[1:][after[:-1]] == [2, 0]).all()
    assert pop.pair_weights == w.tolist()


def test_drawn_pair_frequencies_fit_the_weights():
    K, n = 4, 50000
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    w = np.arange(1, K * K + 1, dtype=np.float64).reshape(K, K)
    w[1, 1] = 0
    w[0, 3] = 0
    thr = torch.from_numpy(pair_thresholds(w, K)).cuda()
    pair = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    obs = np.zeros(K * K)
    for _ in range(4):
        env.assign_pairs(pair, K, thr, counter, seed=42 ^ PAIR_SALT)
        p = _np(pair)
        obs += np.bincount(p[:, 0] * K + p[:, 1], minlength=K * K)
    exp = w.ravel() / w.sum() * obs.sum()
    assert obs[exp == 0].sum() == 0
    chi2 = (((obs - exp) ** 2)[exp > 0] / exp[exp > 0]).sum()
    assert chi2 < 40.0, chi2  # 13 degrees of freedom: p < 2e-4 at this bound


@pytest.mark.parametrize("case", ["cramped_room", "grid_5x5"])
def test_sync_weights_changes_only_the_updated_members_rows(case):
    make, (W, H), _ = CASES[case]
    K, N, T = 3, 240, 20
    models = _models(K, W, H, seed=6)
    pairs = _dev(np.random.RandomState(1).randint(K, size=(N, 2)))
    kw = dict(seed=3, episode_capacity=4)
    pop = SelfPlayRollout(make(N), models, pairs=pairs, **kw)
    ref = SelfPlayRollout(make(N), [copy.deepcopy(m) for m in models], pairs=pairs.clone(), **kw)
    before = pop.collect(T, GAMMA, LAM)
    _equal_batches(before, ref.collect(T, GAMMA, LAM))
    with torch.no_grad():
        for p in models[1].parameters():
            p.mul_(1.5).add_(0.01)
    pop.sync_weights()
    bp, br = pop.collect(T, GAMMA, LAM), ref.collect(T, GAMMA, LAM)
    member_of_row = pairs.view(-1).long()
    other = member_of_row != 1
    # the first transition starts from the same state: rows of members 0 and 2 are unchanged there, member 1's differ
    assert torch.equal(bp.states[0], br.states[0])
    assert torch.equal(bp.logp[0][other], br.logp[0][other]) and torch.equal(bp.values[0][other], br.values[0][other])
    assert not torch.equal(bp.values[0][~other], br.values[0][~other])
