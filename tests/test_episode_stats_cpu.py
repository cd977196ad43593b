"""The episode-statistics restatement (tests/episode_reference.py) against the golden fixtures' events / sparse / shaped
arrays, its reward sum and slot / drop rule, and the ctypes mirror of ovc_episode_stats_t.  No GPU needed."""
import ctypes
import glob
import os
import re

import numpy as np

from episode_reference import EVENT_MASK, EpisodeReference, event_counts, rewards_f32
from helpers import GOLD, Trace
from oracle import cpu
from overcooked_ai_b200 import _native

FIXTURES = sorted(glob.glob(os.path.join(GOLD, "trace_*.npz"))) + [os.path.join(GOLD, "greedy_cramped_room.npz")]


def _replay(tr, factor, capacity=1):
    """Every episode of the fixture as one environment, closed by a done on its last transition.  The event words are the
    CPU oracle's on the fixture's states and actions (the fixture holds bits 0-24; the oracle adds the delivered recipe)."""
    ref = EpisodeReference(tr.layout.deliver_value[None], np.zeros(tr.E, np.int32), capacity)
    sums = np.zeros((tr.E, 2), np.float32)
    for t in range(tr.T):
        st = np.ascontiguousarray(tr.states[:, t])
        _, _, _, ev = cpu.step(tr.tables, tr.starts, st, tr.actions[:, t], horizon=0)
        assert np.array_equal(ev & EVENT_MASK, tr.events[:, t])
        rw = rewards_f32(tr.sparse[:, t], tr.shaped[:, t], factor)
        sums = (sums + rw).astype(np.float32)
        ref.step(tr.shaped[:, t], np.full(tr.E, t == tr.T - 1), ev, np.zeros(tr.E, np.int32), rw)
    return ref, sums


def test_restatement_matches_the_golden_fixtures():
    for path in FIXTURES:
        tr = Trace(path)
        ref, sums = _replay(tr, 0.5)
        fin = ref.finished()
        assert fin["env_index"].tolist() == list(range(tr.E)), tr.name
        assert np.array_equal(fin["ep_game_stats"], event_counts(tr.events & EVENT_MASK).sum(1)), tr.name
        assert np.array_equal(fin["ep_sparse_r_by_agent"], tr.sparse2.sum(1)), tr.name  # deliver_value by recipe == the reference's
        assert np.array_equal(fin["ep_shaped_r_by_agent"], tr.shaped.sum(1)), tr.name
        assert (fin["ep_length"] == tr.T).all() and (fin["layout"] == 0).all() and (fin["partner_seat"] == -1).all()
        assert np.array_equal(fin["ep_reward_by_agent"], sums), tr.name
        assert not ref.event_counts.any() and not ref.ep_length.any() and not ref.sparse.any() and not ref.reward.any()


def test_the_fixtures_fire_every_event_type():
    seen = 0
    for path in FIXTURES:
        seen |= int(np.bitwise_or.reduce(Trace(path).events.reshape(-1) & EVENT_MASK))
    assert seen == EVENT_MASK


def test_reward_sum_is_the_sequential_float32_sum():
    rng = np.random.RandomState(0)
    N, T = 64, 50
    sparse = rng.randint(0, 3, size=(T, N)) * 20
    shaped = rng.randint(0, 4, size=(T, N, 2)) * (rng.rand(T, N, 2) < 0.2)
    factors = rng.rand(T).astype(np.float32) * 1.3
    ref = EpisodeReference(np.zeros((1, 16)), np.zeros(N, np.int32), 1)
    rw = np.stack([rewards_f32(sparse[t], shaped[t], factors[t]) for t in range(T)])
    for t in range(T):
        ref.step(shaped[t], np.zeros(N), np.zeros((N, 2), np.int32), np.zeros(N, np.int32), rw[t])
    assert np.array_equal(ref.reward, np.cumsum(rw, axis=0, dtype=np.float32)[-1])
    assert np.array_equal(rw[3], np.float32(sparse[3])[:, None] + factors[3] * np.float32(shaped[3]))


def test_slots_and_drops():
    """Slot k of env e is its k-th episode since clear(); past the capacity episodes are counted, not written."""
    N, cap = 3, 2
    ref = EpisodeReference(np.arange(32).reshape(2, 16), np.array([0, 1, 1], np.int32), cap)
    ev = np.zeros((N, 2), np.int64)
    ev[:, 1] = (1 << 15) | (5 << 25)  # agent 1 delivers recipe 5 every transition
    ends = {0: [0, 1, 2], 1: [2], 2: [0, 2, 4, 6]}
    lid = np.array([0, 1, 1], np.int32)
    for t in range(7):
        done = np.array([t in ends[e] for e in range(N)])
        lid = np.where(done, [1, 1, 1 - lid[2]], lid).astype(np.int32)  # a reset draws the next episode's layout
        ref.step(np.ones((N, 2), np.int32), done, ev, lid, np.ones((N, 2), np.float32), np.array([0, -1, 1]))
    assert ref.count.tolist() == [2, 1, 2] and ref.dropped.tolist() == [1, 0, 2]
    fin = ref.finished()
    assert fin["env_index"].tolist() == [0, 1, 2, 0, 2]  # (slot, env) order
    assert fin["ep_length"].tolist() == [1, 3, 1, 1, 2]
    # a delivery on an episode's last transition is credited to the layout it was played on, not the next one's
    assert fin["layout"].tolist() == [0, 1, 1, 1, 0] and fin["ep_sparse_r_by_agent"][:, 1].tolist() == [5, 63, 21, 21, 10]
    assert fin["partner_seat"].tolist() == [0, -1, 1, 0, 1]
    assert ref.ep_length.tolist() == [4, 4, 0]


def test_descriptor_matches_the_header():
    """EpisodeStatsDesc lists ovc_episode_stats_t's fields in the header's order, at its 160 bytes."""
    hdr = open(os.path.join(os.path.dirname(_native.__file__), "..", "include", "ovc_b200.h")).read()
    body = re.search(r"typedef struct ovc_episode_stats \{(.*?)\} ovc_episode_stats_t;", hdr, re.S).group(1)
    fields = re.findall(r"(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert fields == [f for f, _ in _native.EpisodeStatsDesc._fields_]
    assert ctypes.sizeof(_native.EpisodeStatsDesc) == 160
    assert "ovc_record_transition_stats" in _native.EXPORTED_SYMBOLS
