"""Finished episodes on the device (ovc_record_transition_stats, EpisodeStats / EpisodeRecords, SelfPlayRollout's
episodes), bit for bit against the restatement in tests/episode_reference.py fed by the CPU oracle."""
import math

import numpy as np
import pytest
import torch

from episode_reference import EVENT_MASK, RECORD_KEYS, EpisodeReference, event_counts, rewards_f32
from helpers import GOLD, TRACE_FILES, Trace
from oracle import cpu
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeRecords, EpisodeStats
from overcooked_ai_b200.selfplay import BCPolicy, RllibShapedCNN, SelfPlayRollout

pytestmark = pytest.mark.gpu

SENTINEL = -7


def _np(t):
    return t.cpu().numpy()


def _with_tails(obj, names, pad=67):
    """Replace obj's tensors ``names`` by views at the front of larger buffers whose tails hold a sentinel; returns the
    (buffer, numel) pairs to check later."""
    tails = []
    for n in names:
        t = getattr(obj, n)
        buf = torch.full((t.numel() + pad,), SENTINEL, dtype=t.dtype, device=t.device)
        buf[:t.numel()].copy_(t.view(-1))
        setattr(obj, n, buf[:t.numel()].view(t.shape))
        tails.append((buf, t.numel()))
    return tails


def _check_equal(stats, rec, ref):
    for got, want in zip(stats.state_tensors(), ref.running()):
        assert np.array_equal(_np(got), want)
    assert np.array_equal(_np(rec.count), ref.count) and np.array_equal(_np(rec.dropped), ref.dropped)
    fin, want = rec.finished(), ref.finished()
    assert set(fin) == set(want)
    for k in want:
        assert np.array_equal(_np(fin[k]), want[k]), k


CASES = {  # layouts, mdp params, random_layout
    "mixed": (["cramped_room", "asymmetric_advantages", "coordination_ring"], {}, False),
    "bonus_order": (["bonus_order_test"], {}, False),
    "old_dynamics": (["cramped_room"], {"old_dynamics": True}, False),
    "random_layout": (["cramped_room", "cramped_room_tomato", "marshmallow_experiment"], {}, True),
}


@pytest.mark.parametrize("capacity", [5, 2])
@pytest.mark.parametrize("case", sorted(CASES))
def test_stats_kernel_vs_reference(case, capacity):
    """Random interact-biased play from random starts, horizon 7 over 30 transitions (several episodes per env), N = 1037
    (not a multiple of the block), a factor that changes every transition, random partner seats; capacity 5 holds every
    episode, capacity 2 drops.  Every output buffer has a sentinel tail that must stay untouched."""
    names, params, random_layout = CASES[case]
    layouts = [L.compile_layout(n, **params) for n in names]
    n, H, T = 1037, 7, 30
    # random starts with objects (held soups among them) so that short episodes deliver
    env = BatchedOvercookedEnv(layouts, n, horizon=H, auto_reset=True, random_layout=random_layout, random_start_pos=True,
                               rnd_obj_prob_thresh=0.6, seed=3)
    vals = np.stack([l.deliver_value for l in layouts])
    if random_layout:
        assert len({tuple(v) for v in vals}) == len(layouts)
    rs = cpu.random_start(3, 0.6, True, random_layout)
    ref_state = _np(env.state).copy()
    stats, rec = EpisodeStats(env), EpisodeRecords(env, capacity)
    tails = _with_tails(stats, ["event_counts", "cumulative_sparse_rewards_by_agent", "cumulative_shaped_rewards_by_agent",
                                "ep_reward_by_agent", "ep_length", "layout_id"])
    tails += _with_tails(rec, ["length", "layout", "partner_seat", "sparse_r_by_agent", "shaped_r_by_agent", "game_stats",
                               "reward_by_agent", "_counters"])
    rec.count, rec.dropped = rec._counters[0], rec._counters[1]
    ref = EpisodeReference(vals, ref_state[:, 3] & 0xFF, capacity)
    rng = np.random.RandomState(len(case) + capacity)
    factor = torch.zeros(1, dtype=torch.float32, device="cuda")
    rewards = torch.zeros((n, 2), dtype=torch.float32, device="cuda")
    seats = rng.randint(-1, 2, size=n).astype(np.int32)
    d_seats = torch.from_numpy(seats).cuda()
    delivered = 0
    for t in range(T):
        a = rng.randint(0, 6, size=(n, 2)).astype(np.int32)
        a[rng.rand(n, 2) < 0.4] = 5
        f = float(np.float32(rng.rand() * 1.5))
        factor.fill_(f)
        env.step(torch.from_numpy(a).cuda())
        env.record_transition(factor, rewards=rewards, stats=stats, records=rec, partner_seat=d_seats)
        sp, sh, dn, ev = cpu.step(env._tab_host, env._starts_host, ref_state, a, horizon=H, flags=1, rs=rs)
        rw = rewards_f32(sp, sh, f)
        assert np.array_equal(_np(rewards), rw)
        ref.step(sh, dn, ev, ref_state[:, 3] & 0xFF, rw, seats)
        delivered += int(((ev >> 15) & 1).sum())
    assert np.array_equal(_np(env.state), ref_state)
    _check_equal(stats, rec, ref)
    assert delivered > 0 and (ref.count == min(capacity, T // H)).all()
    assert (ref.dropped > 0).any() == (capacity < T // H)
    for buf, k in tails:
        assert (_np(buf[k:]) == SENTINEL).all()
    if random_layout:
        fin = ref.finished()
        assert len(np.unique(fin["layout"])) == len(layouts) and (fin["ep_sparse_r"] > 0).any()


@pytest.mark.parametrize("path", TRACE_FILES + [GOLD + "/greedy_cramped_room.npz"], ids=lambda p: p.split("/")[-1][:-4])
def test_golden_traces_counts(path):
    """Every fixture replayed through env.step + the stats kernel: the running counts are the fixture's event bits, the
    sums its per-agent rewards."""
    tr = Trace(path)
    env = BatchedOvercookedEnv(tr.layout, tr.E, horizon=0)
    env.state.copy_(torch.from_numpy(np.ascontiguousarray(tr.states[:, 0])).cuda())
    stats, rec = EpisodeStats(env), EpisodeRecords(env, 1)
    one = torch.ones(1, dtype=torch.float32, device="cuda")
    acts = torch.from_numpy(np.ascontiguousarray(tr.actions.transpose(1, 0, 2))).cuda()
    for t in range(tr.T):
        env.step(acts[t])
        env.record_transition(one, stats=stats, records=rec)
    assert np.array_equal(_np(stats.event_counts), event_counts(tr.events & EVENT_MASK).sum(1))
    assert np.array_equal(_np(stats.cumulative_sparse_rewards_by_agent), tr.sparse2.sum(1))
    assert np.array_equal(_np(stats.cumulative_shaped_rewards_by_agent), tr.shaped.sum(1))
    assert (_np(stats.ep_length) == tr.T).all() and not rec.count.any() and not rec.dropped.any()


def _replay_window(env, b, ref, H):
    """Feed ``ref`` the oracle's replay of the window from b.states[t] / b.actions[t]; checks the states follow it."""
    T, N = b.dones.shape
    st, ac, rw = _np(b.states), _np(b.actions), _np(b.rewards)
    ps = None if b.partner_seat is None else _np(b.partner_seat).astype(np.int32)
    state = st[0].copy()
    ref.clear()
    for t in range(T):
        assert np.array_equal(st[t], state), t
        _, sh, dn, ev = cpu.step(env._tab_host, env._starts_host, state, ac[t].reshape(N, 2), horizon=H, flags=1)
        ref.step(sh, dn, ev, state[:, 3] & 0xFF, rw[t].reshape(N, 2), None if ps is None else ps[t])
    assert np.array_equal(_np(env.state), state)


def _records_equal(a, b):
    for k in RECORD_KEYS + ("count", "dropped"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.parametrize("H", [13, 400])
@pytest.mark.parametrize("T", [7, 150, 400])
def test_collect_episodes_vs_oracle_replay(T, H):
    """collect(), graph and eager: b.episodes and the running state equal the restatement fed by the oracle's replay of
    batch.states / batch.actions, over three windows whose episodes cross window boundaries, with the shaping factor
    changed between windows; ep_reward_by_agent is the float32 sum of batch.rewards over each episode."""
    n, seed = 300, 4
    torch.manual_seed(1)
    model = RllibShapedCNN(5, 4).cuda()
    envs = [BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True) for _ in range(2)]
    pre = H - 5 if T < H else 3
    for e in envs:
        e.rollout(torch.full((pre, n, 2), 4, dtype=torch.int32, device="cuda"))  # mid-episode, windows not aligned with ends
    sps = [SelfPlayRollout(e, model=model, use_graph=g, seed=seed) for e, g in zip(envs, (True, False))]
    ref = EpisodeReference(envs[0].layouts[0].deliver_value[None], np.zeros(n, np.int32), math.ceil(T / H))
    ended = 0
    for w, f in enumerate((1.0, 0.375, 0.0)):
        for sp in sps:
            sp.reward_shaping_factor = f
        bs = [sp.collect(T, 0.99, 0.95) for sp in sps]
        assert bs[0].episodes.capacity == math.ceil(T / H)
        _records_equal(bs[0].episodes, bs[1].episodes)
        for x, y in zip(sps[0].stats.state_tensors(), sps[1].stats.state_tensors()):
            assert torch.equal(x, y)
        _replay_window(envs[0], bs[0], ref, H)
        _check_equal(sps[0].stats, bs[0].episodes, ref)
        assert not ref.dropped.any()
        ended += int(ref.count.sum())
    assert ended > 0


def test_partner_seat_of_each_record():
    """With a BC partner at bc_factor 0.5 every record's partner_seat is batch.partner_seat on that episode's
    transitions."""
    n, H, T = 512, 13, 60
    torch.manual_seed(2)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True)
    sp = SelfPlayRollout(env, model=RllibShapedCNN(5, 4).cuda(), seed=8, partner=BCPolicy().cuda(), bc_factor=0.5)
    ref = EpisodeReference(env.layouts[0].deliver_value[None], np.zeros(n, np.int32), math.ceil(T / H))
    for _ in range(2):
        b = sp.collect(T, 0.99, 0.95)
        _replay_window(env, b, ref, H)
        _check_equal(sp.stats, b.episodes, ref)
        fin = {k: _np(v) for k, v in b.episodes.finished().items()}
        ps, dn = _np(b.partner_seat).astype(np.int32), _np(b.dones).astype(np.int64)
        assert set(fin["partner_seat"].tolist()) == {-1, 0, 1}
        # slot k of env e is its k-th done in the window: check it exactly
        k_of = np.cumsum(dn, 0) - 1
        for t, e in zip(*np.nonzero(dn)):
            assert _np(b.episodes.partner_seat)[k_of[t, e], e] == ps[t, e]


def test_run_and_collect_leave_the_same_records():
    """run() and collect() from the same seed leave the same records and running state; graph capture leaves the running
    state and the records unchanged."""
    n, T, H, seed = 300, 40, 13, 5
    torch.manual_seed(3)
    model = RllibShapedCNN(5, 4).cuda()
    envs = [BatchedOvercookedEnv("cramped_room", n, horizon=H, auto_reset=True) for _ in range(2)]
    for e in envs:
        e.rollout(torch.zeros((3, n, 2), dtype=torch.int32, device="cuda"))
    cap = math.ceil(T / H)
    sp_run = SelfPlayRollout(envs[0], model=model, seed=seed, episode_capacity=cap)
    sp_col = SelfPlayRollout(envs[1], model=model, seed=seed)
    sp_run.run(2)
    sp_run.episodes.clear()
    sp_run.stats.ep_length.fill_(9)  # a recognisable running state before the capture
    before = [t.clone() for t in sp_run.stats.state_tensors() + sp_run.episodes.tensors()]
    sp_run.graph = None
    sp_run.run(0)  # capture only
    assert sp_run.graph is not None
    for x, y in zip(before, sp_run.stats.state_tensors() + sp_run.episodes.tensors()):
        assert torch.equal(x, y)
    sp_run.stats.ep_length.fill_(0)
    # the two rollouts from the same state, running state and draw counter
    envs[1].state.copy_(envs[0].state)
    sp_col._draw_counter.copy_(sp_run._draw_counter)
    for x, y in zip(sp_col.stats.state_tensors(), sp_run.stats.state_tensors()):
        x.copy_(y)
    sp_run.run(T)
    b = sp_col.collect(T, 0.99, 0.95)
    assert torch.equal(envs[0].state, envs[1].state)
    _records_equal(sp_run.episodes, b.episodes)
    assert int(b.episodes.count.sum()) > 0
    for x, y in zip(sp_col.stats.state_tensors(), sp_run.stats.state_tensors()):
        assert torch.equal(x, y)
