"""A population of self-play learners on the device: ovc_encode_linear_grouped, ovc_wide_layers_grouped and
ovc_policy_tail_grouped against ovc_encode_linear, ovc_wide_layers and ovc_policy_tail_logp per member (distinct random
weights, uneven blocks that are not tile aligned, sentinels past the end, the counter advanced once), and
SelfPlayRollout with a list model against one SelfPlayRollout per member, block by block, bit for bit, in run() and over
collect() windows whose episodes cross the window boundary, on every path the population takes (K7 -> K9 -> K8, K9 grouped at 4 members and per member at 1 and 3; K7 ->
library layers -> draw kernel on a 5x5 grid; K2 -> library layers -> grouped K8 on a pool of 9 layouts), with random
starts, use_phi and sync_weights."""
import numpy as np
import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import RllibShapedCNN, SelfPlayRollout
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95
SENTINEL = -7


def _np(t):
    return t.cpu().numpy()


# ------------------------------------------------------------------------------------------------ the grouped K8


def _tables(rng, K, k0, n_hidden):
    bf = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda().to(torch.bfloat16)
    f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    nh = max(n_hidden, 1)
    return (bf(rng.normal(size=(K, 64, k0)) / np.sqrt(k0)), f32(rng.normal(size=(K, 64)) * 0.1),
            bf(rng.normal(size=(K, nh, 64, 64)) / 8), f32(rng.normal(size=(K, nh, 64)) * 0.1),
            bf(rng.normal(size=(K, 8, 64)) / 4), f32(rng.normal(size=(K, 8)) * 0.1))


def _tail_outputs(n, pad, logp):
    """actions, values, scores and (optionally) logp, each with ``pad`` sentinel rows past the ``n`` rows."""
    out = [torch.full((n + pad,), SENTINEL, dtype=torch.int32, device="cuda"),
           torch.full((n + pad,), float(SENTINEL), device="cuda"), torch.full((n + pad, 8), float(SENTINEL), device="cuda")]
    return out + [torch.full((n + pad,), float(SENTINEL), device="cuda") if logp else None]


BLOCKS = {1: [4096], 3: [1, 7, 129], 64: None}  # environments per member; K = 64: 1, 7, 129, 4096 and 60 random sizes


@pytest.mark.parametrize("logp", [True, False], ids=["logp", "plain"])
@pytest.mark.parametrize("k0,n_hidden", [(160, 2), (64, 0), (256, 3)])
@pytest.mark.parametrize("K", [1, 3, 64])
def test_grouped_tail_equals_the_tail_of_each_member(K, k0, n_hidden, logp):
    lib = _native.lib()
    rng = np.random.RandomState(K * 1000 + k0 + n_hidden)
    blocks = BLOCKS[K] or [1, 7, 129, 4096] + rng.randint(1, 300, size=60).tolist()
    offs = np.concatenate([[0], np.cumsum(blocks)]) * 2  # two rows per environment
    n, pad = int(offs[-1]), 37
    x = torch.from_numpy(rng.normal(size=(n, k0)).astype(np.float32)).cuda().to(torch.bfloat16)
    w1, b1, wh, bh, wo, bo = _tables(rng, K, k0, n_hidden)
    seed = 0x1234_5678_9ABC_DEF0 + K
    counter = torch.tensor([41, 0], dtype=torch.int64, device="cuda")
    acts, vals, scores, lp = _tail_outputs(n, pad, logp)
    offsets = torch.from_numpy(offs.astype(np.int32)).cuda()
    _native.check(lib.ovc_policy_tail_grouped(
        x.data_ptr(), n, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), n_hidden, wo.data_ptr(), bo.data_ptr(),
        0.3, 6, seed, counter.data_ptr(), offsets.data_ptr(), K, acts.data_ptr(), vals.data_ptr(), scores.data_ptr(),
        0 if lp is None else lp.data_ptr(), None))
    assert _np(counter).tolist() == [42, 0], "the step advances exactly once per launch"
    for k in range(K):
        a, b = int(offs[k]), int(offs[k + 1])
        c = torch.tensor([41, 0], dtype=torch.int64, device="cuda")
        ra, rv, rs, rl = _tail_outputs(n, 0, True)
        _native.check(lib.ovc_policy_tail_logp(
            x.data_ptr(), n, k0, 0.2, w1[k].data_ptr(), b1[k].data_ptr(), wh[k].data_ptr(), bh[k].data_ptr(), n_hidden, wo[k].data_ptr(),
            bo[k].data_ptr(), 0.3, 6, seed, c.data_ptr(), ra.data_ptr(), rv.data_ptr(), rs.data_ptr(), rl.data_ptr(), None))
        assert torch.equal(acts[a:b], ra[a:b]) and torch.equal(vals[a:b], rv[a:b]) and torch.equal(scores[a:b], rs[a:b]), k
        if lp is not None:
            assert torch.equal(lp[a:b], rl[a:b]), k
    assert (_np(acts[n:]) == SENTINEL).all() and (_np(vals[n:]) == SENTINEL).all() and (_np(scores[n:]) == SENTINEL).all()
    if lp is not None:
        assert (_np(lp[n:]) == SENTINEL).all()
    assert len(np.unique(_np(acts[:n]))) == 6


def test_grouped_tail_leaves_rows_outside_every_block_and_empty_blocks_alone():
    lib = _native.lib()
    rng = np.random.RandomState(5)
    K, k0, n = 4, 160, 500
    offs = np.array([10, 10, 100, 100, 480], np.int32)  # rows [0, 10) and [480, 500) belong to no member; members 0 and 2 are empty
    x = torch.from_numpy(rng.normal(size=(n, k0)).astype(np.float32)).cuda().to(torch.bfloat16)
    w1, b1, wh, bh, wo, bo = _tables(rng, K, k0, 2)
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    acts, vals, scores, lp = _tail_outputs(n, 0, True)
    _native.check(lib.ovc_policy_tail_grouped(
        x.data_ptr(), n, k0, 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), 2, wo.data_ptr(), bo.data_ptr(), 0.3, 6, 9,
        counter.data_ptr(), torch.from_numpy(offs).cuda().data_ptr(), K, acts.data_ptr(), vals.data_ptr(), scores.data_ptr(),
        lp.data_ptr(), None))
    assert _np(counter).tolist() == [1, 0]
    for r in (slice(0, 10), slice(480, n)):
        assert (_np(acts[r]) == SENTINEL).all() and (_np(vals[r]) == SENTINEL).all() and (_np(lp[r]) == SENTINEL).all()
        assert (_np(scores[r]) == SENTINEL).all()
    assert (_np(acts[10:480]) != SENTINEL).all()


@pytest.mark.parametrize("K", [1, 3, 64])
def test_grouped_encode_linear_equals_the_encoding_of_each_member(K):
    lib = _native.lib()
    rng = np.random.RandomState(K + 11)
    blocks = BLOCKS[K] or [1, 7, 129, 4096] + rng.randint(1, 300, size=60).tolist()
    offs = np.concatenate([[0], np.cumsum(blocks)]).astype(np.int32)
    n, n_out = int(offs[-1]), 512
    env = BatchedOvercookedEnv("cramped_room", n, horizon=15, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=K)
    env.reset()
    wt = (torch.randn(K, 520, n_out, device="cuda") * 0.2).to(torch.bfloat16)
    bias = torch.randn(K, n_out, device="cuda") * 0.1
    out = torch.full((2 * n + 5, n_out), float("nan"), dtype=torch.bfloat16, device="cuda")
    _native.check(lib.ovc_encode_linear_grouped(env.tables.data_ptr(), env.n_layouts, env.state.data_ptr(), wt.data_ptr(), bias.data_ptr(),
                                                torch.from_numpy(offs).cuda().data_ptr(), K, out.data_ptr(), n, env.state_words, 5, 4, 15,
                                                n_out, 0.2, None))
    for k in range(K):
        want = env.encoded_linear(wt[k].contiguous(), bias[k].contiguous())
        assert torch.equal(out[2 * offs[k]:2 * offs[k + 1]], want[2 * offs[k]:2 * offs[k + 1]]), k
    assert torch.isnan(out[2 * n:].float()).all()


@pytest.mark.parametrize("K", [1, 3, 64])
def test_grouped_wide_layers_equal_the_wide_layers_of_each_member(K):
    lib = _native.lib()
    rng = np.random.RandomState(K + 21)
    blocks = BLOCKS[K] or [1, 7, 129, 4096] + rng.randint(1, 300, size=60).tolist()
    offs = (np.concatenate([[0], np.cumsum(blocks)]) * 2).astype(np.int32)  # rows
    m = int(offs[-1])
    a0 = (torch.randn(m, 512, device="cuda") * 0.5).to(torch.bfloat16)
    w1 = (torch.randn(K, 512, 512, device="cuda") / 22).to(torch.bfloat16)
    w2 = (torch.randn(K, 160, 512, device="cuda") / 22).to(torch.bfloat16)
    b1, b2 = torch.randn(K, 512, device="cuda") * 0.1, torch.randn(K, 160, device="cuda") * 0.1
    z = torch.full((m + 130, 160), float("nan"), dtype=torch.bfloat16, device="cuda")
    _native.check(lib.ovc_wide_layers_grouped(a0.data_ptr(), m, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(), 160, 0.2,
                                              torch.from_numpy(offs).cuda().data_ptr(), K, z.data_ptr(), None))
    for k in range(K):
        want = torch.empty((m, 160), dtype=torch.bfloat16, device="cuda")
        _native.check(lib.ovc_wide_layers(a0.data_ptr(), m, 512, w1[k].data_ptr(), b1[k].data_ptr(), 512, w2[k].data_ptr(), b2[k].data_ptr(),
                                          160, 0.2, want.data_ptr(), None))
        assert torch.equal(z[offs[k]:offs[k + 1]], want[offs[k]:offs[k + 1]]), k
    assert torch.isnan(z[m:].float()).all()


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
    "pool_9": (lambda n: BatchedOvercookedEnv(POOL_5X4, n, horizon=10, auto_reset=True, env_layout=np.arange(n) % 9),
               (5, 4), (False, False, True)),
}


def _block_equal(pop, singles, offs, bp=None, bss=None):
    """Block k of the population (its live state, or the batch bp) equals single k (or its batch bss[k]) on that block."""
    for k, s in enumerate(singles):
        a, b = offs[k], offs[k + 1]
        if bp is None:
            assert torch.equal(pop.env.state[a:b], s.env.state[a:b]), k
            assert torch.equal(pop.actions[a:b], s.actions[a:b]) and torch.equal(pop.values[a:b], s.values[a:b]), k
            assert torch.equal(pop.ret_sparse[a:b], s.ret_sparse[a:b]) and torch.equal(pop.ret_mixed[a:b], s.ret_mixed[a:b]), k
            fp, fs = pop.episodes.finished(), s.episodes.finished()
        else:
            bs = bss[k]
            for f in ("actions", "logp", "values", "rewards", "advantages", "value_targets"):
                assert torch.equal(getattr(bp, f)[:, 2 * a:2 * b], getattr(bs, f)[:, 2 * a:2 * b]), (k, f)
            assert torch.equal(bp.states[:, a:b], bs.states[:, a:b]) and torch.equal(bp.dones[:, a:b], bs.dones[:, a:b]), k
            assert torch.equal(bp.last_values[2 * a:2 * b], bs.last_values[2 * a:2 * b]), k
            fp, fs = bp.episodes.finished(), bs.episodes.finished()
        ip = (fp["env_index"] >= a) & (fp["env_index"] < b)
        is_ = (fs["env_index"] >= a) & (fs["env_index"] < b)
        assert int(is_.sum()) > 0, "premise: episodes end in every block"
        for f in fs:
            assert torch.equal(fp[f][ip], fs[f][is_]), (k, f)


def _rollouts(case, K, blocks, graph, use_phi=False, n=None):
    make, (W, H), flags = CASES[case]
    n = n or sum(blocks)
    models = _models(K, W, H, seed=len(case))
    kw = dict(seed=77, use_graph=graph, use_phi=use_phi, episode_capacity=4)
    pop = SelfPlayRollout(make(n), models, blocks=blocks, **kw)
    singles = [SelfPlayRollout(make(n), m, **kw) for m in models]
    assert (pop.fused_first_layer, pop.fused_wide, pop.fused_tail) == flags
    assert all((s.fused_first_layer, s.fused_wide, s.fused_tail) == flags for s in singles)
    return pop, singles, models


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", list(CASES))
def test_each_block_of_collect_and_run_equals_the_members_own_selfplay(case, graph):
    blocks = [1, 7, 129, 300 - 137]
    pop, singles, _ = _rollouts(case, 4, blocks, graph)
    offs = _np(pop.blocks).tolist()
    assert offs == [0, 1, 8, 137, 300]
    assert torch.equal(pop.member, torch.repeat_interleave(torch.arange(4, device="cuda"), torch.tensor(blocks, device="cuda")).int())
    for w in range(2):  # two windows: episodes cross the boundary
        bp = pop.collect(25, GAMMA, LAM)
        bss = [s.collect(25, GAMMA, LAM) for s in singles]
        _block_equal(pop, singles, offs, bp, bss)
    for s in [pop] + singles:
        s.episodes.clear()
    pop.run(30)
    for s in singles:
        s.run(30)
    _block_equal(pop, singles, offs)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_use_phi_blocks_equal_the_members_own_selfplay(graph):
    pop, singles, _ = _rollouts("cramped_room", 3, None, graph, use_phi=True, n=301)  # equal blocks: 100, 100, 101
    offs = _np(pop.blocks).tolist()
    assert offs == [0, 100, 200, 301]
    for w in range(2):
        bp = pop.collect(24, GAMMA, LAM)
        _block_equal(pop, singles, offs, bp, [s.collect(24, GAMMA, LAM) for s in singles])


@pytest.mark.parametrize("case", ["cramped_room", "pool_9"])
def test_one_member_equals_selfplay_on_every_output(case):
    pop, (single,), _ = _rollouts(case, 1, [300], True)
    for w in range(2):
        bp, bs = pop.collect(20, GAMMA, LAM), single.collect(20, GAMMA, LAM)
        for f in ("states", "actions", "logp", "values", "rewards", "dones", "advantages", "value_targets", "last_values"):
            assert torch.equal(getattr(bp, f), getattr(bs, f)), f
        fp, fs = bp.episodes.finished(), bs.episodes.finished()
        assert all(torch.equal(fp[f], fs[f]) for f in fs) and len(fs["env_index"]) > 0
    pop.run(15), single.run(15)
    assert torch.equal(pop.env.state, single.env.state) and torch.equal(pop.actions, single.actions)
    assert torch.equal(pop.values, single.values) and torch.equal(pop.ret_mixed, single.ret_mixed)


@pytest.mark.parametrize("case", ["cramped_room", "random_starts", "grid_5x5", "pool_9"])
def test_sync_weights_changes_one_members_block_only(case):
    pop, singles, models = _rollouts(case, 3, [50, 77, 73], True)
    offs = _np(pop.blocks).tolist()
    before = [b.clone() for b in pop._learners._tail_stack] if pop.fused_tail else None
    _block_equal(pop, singles, offs, pop.collect(20, GAMMA, LAM), [s.collect(20, GAMMA, LAM) for s in singles])
    with torch.no_grad():  # member 1 after a "learner update"; single 1 shares the module
        for p in models[1].parameters():
            p.mul_(1.5).add_(0.01)
    pop.sync_weights()
    singles[1].sync_weights()
    if before is not None:  # the stacked tables changed in member 1's entry only
        for old, new in zip(before, pop._learners._tail_stack):
            assert torch.equal(old[0], new[0]) and torch.equal(old[2], new[2]) and not torch.equal(old[1], new[1])
    bp = pop.collect(20, GAMMA, LAM)
    bss = [s.collect(20, GAMMA, LAM) for s in singles]
    _block_equal(pop, singles, offs, bp, bss)
    # the new weights are in use: member 1's block is not what its old weights would draw
    fresh = SelfPlayRollout(CASES[case][0](200), _models(3, *CASES[case][1], seed=len(case))[1], seed=77, episode_capacity=4)
    fresh.collect(20, GAMMA, LAM)
    assert not torch.equal(fresh.collect(20, GAMMA, LAM).logp[:, 2 * offs[1]:2 * offs[2]], bp.logp[:, 2 * offs[1]:2 * offs[2]])
