"""numpy restatement of the episode statistics of ovc_record_transition_stats (include/ovc_b200.h): the running state, the
float32 reward sums and the record slots with their drop rule.  Fed transition by transition with ovc_step's outputs."""
import numpy as np

N_EVENTS = 25
EVENT_MASK = (1 << N_EVENTS) - 1
SOUP_DELIVERY = 15
RECIPE_SHIFT = 25

RECORD_KEYS = ("length", "layout", "partner_seat", "sparse_r_by_agent", "shaped_r_by_agent", "game_stats", "reward_by_agent")


def event_counts(events):
    """int32 [..., 25]: bit b < 25 of every event word, as 0 / 1."""
    return ((np.asarray(events)[..., None] >> np.arange(N_EVENTS)) & 1).astype(np.int32)


def rewards_f32(sparse, shaped, factor):
    """rewards[e][i] = float32(sparse[e]) + float32(factor) * float32(shaped[e][i]), the product rounded first."""
    sp = np.asarray(sparse).astype(np.float32)[:, None]
    return (sp + np.float32(factor) * np.asarray(shaped).astype(np.float32)).astype(np.float32)


class EpisodeReference(object):
    """The kernel's definition for N environments: ``step`` folds one transition in, ``finished`` lists the records in
    (slot, env) order as ``EpisodeRecords.finished`` does."""

    def __init__(self, deliver_value, layout_id, capacity, members=False, pairs=False):
        self.members, self.pairs = bool(members), bool(pairs)
        self.deliver_value = np.asarray(deliver_value, dtype=np.int64).reshape(-1, 16)
        self.layout_id = np.array(layout_id, dtype=np.int32)
        N = len(self.layout_id)
        self.capacity = int(capacity)
        self.event_counts = np.zeros((N, 2, N_EVENTS), np.int32)
        self.sparse = np.zeros((N, 2), np.int64)
        self.shaped = np.zeros((N, 2), np.int64)
        self.reward = np.zeros((N, 2), np.float32)
        self.ep_length = np.zeros(N, np.int32)
        self.clear()

    def clear(self):
        N, C = len(self.layout_id), self.capacity
        self.count = np.zeros(N, np.int32)
        self.dropped = np.zeros(N, np.int32)
        self.records = {"length": np.zeros((C, N), np.int32), "layout": np.zeros((C, N), np.int32),
                        "partner_seat": np.zeros((C, N), np.int32), "sparse_r_by_agent": np.zeros((C, N, 2), np.int64),
                        "shaped_r_by_agent": np.zeros((C, N, 2), np.int64), "game_stats": np.zeros((C, N, 2, N_EVENTS), np.int32),
                        "reward_by_agent": np.zeros((C, N, 2), np.float32)}
        if self.members:
            self.records["partner_member"] = np.zeros((C, N), np.int32)
        if self.pairs:
            self.records["pair"] = np.zeros((C, N, 2), np.int32)

    def save_records(self):
        """The record set (records, count, dropped, capacity), to be put back by ``load_records``: a rollout keeps run()'s
        records and each window's apart while the running state is shared."""
        return self.records, self.count, self.dropped, self.capacity

    def load_records(self, saved):
        self.records, self.count, self.dropped, self.capacity = saved

    def empty_records(self, capacity):
        kept = self.save_records()
        self.capacity = int(capacity)
        self.clear()
        fresh = self.save_records()
        self.load_records(kept)
        return fresh

    def step(self, shaped, done, events, new_layout_id, rewards, partner_seat=None, member=None, pair=None):
        """shaped [N,2], done [N], events [N,2] of one ovc_step; new_layout_id [N] = word 3 & 0xFF of the records after it;
        rewards float32 [N,2] (``rewards_f32``); partner_seat [N] or None (-1 in every record); member [N] / pair [N, 2]: the
        ending episodes' member / pair (recorded with ``members`` / ``pairs``)."""
        events = np.asarray(events).astype(np.int64)
        rec = (events >> RECIPE_SHIFT) & 15
        delivered = (events >> SOUP_DELIVERY) & 1
        self.sparse += self.deliver_value[self.layout_id[:, None], rec] * delivered
        self.shaped += np.asarray(shaped)
        self.ep_length += 1
        self.event_counts += event_counts(events & EVENT_MASK)
        self.reward = (self.reward + np.asarray(rewards, dtype=np.float32)).astype(np.float32)
        ended_layout = self.layout_id.copy()
        self.layout_id = np.asarray(new_layout_id, dtype=np.int32).copy()
        for e in np.nonzero(np.asarray(done) != 0)[0]:
            k = self.count[e]
            if k < self.capacity:
                r = self.records
                r["length"][k, e], r["layout"][k, e] = self.ep_length[e], ended_layout[e]
                r["partner_seat"][k, e] = -1 if partner_seat is None else partner_seat[e]
                r["sparse_r_by_agent"][k, e], r["shaped_r_by_agent"][k, e] = self.sparse[e], self.shaped[e]
                r["game_stats"][k, e], r["reward_by_agent"][k, e] = self.event_counts[e], self.reward[e]
                if self.members:
                    r["partner_member"][k, e] = member[e]
                if self.pairs:
                    r["pair"][k, e] = pair[e]
                self.count[e] = k + 1
            else:
                self.dropped[e] += 1
            self.sparse[e] = self.shaped[e] = 0
            self.reward[e] = 0
            self.event_counts[e] = 0
            self.ep_length[e] = 0

    def finished(self):
        k, e = np.nonzero(np.arange(self.capacity)[:, None] < self.count[None, :])
        r = self.records
        out = {"env_index": e, "ep_game_stats": r["game_stats"][k, e], "ep_sparse_r_by_agent": r["sparse_r_by_agent"][k, e],
               "ep_shaped_r_by_agent": r["shaped_r_by_agent"][k, e], "ep_sparse_r": r["sparse_r_by_agent"][k, e].sum(1),
               "ep_shaped_r": r["shaped_r_by_agent"][k, e].sum(1), "ep_length": r["length"][k, e],
               "ep_reward_by_agent": r["reward_by_agent"][k, e], "layout": r["layout"][k, e], "partner_seat": r["partner_seat"][k, e]}
        for key in ("partner_member", "pair"):
            if key in r:
                out[key] = r[key][k, e]
        return out

    def running(self):
        """The running state in the order of ``EpisodeStats.state_tensors``."""
        return [self.event_counts, self.sparse, self.shaped, self.reward, self.ep_length, self.layout_id]
