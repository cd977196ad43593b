"""The rollout driver (``SelfPlayRollout`` / ``AgentPairRollout`` with ``_NetworkAgent``, ``_BCAgent``, ``_Population`` and
``_Learners``) restated sequentially on the host, from the documented contracts (DESIGN §4, the docstrings of selfplay.py):
which agent holds each row, which Philox key and counter each draw uses, when the per-episode draws happen, what goes into
the rewards, the returns, the records and the sample batch.  It uses the C oracle, float64 forwards of the models and numpy
only: no rollout class, no environment method, no native library.  The per-kernel restatements it is built from are here
too, so that each is stated once: the seat, member and pair draws, ``ovc_learner_rows``, the BC network on
``featurize_state`` and GAE on one row per environment; the greedy agent is tests/greedy_reference.py's.

Each agent is evaluated on the rows it holds and nothing else; there is no grouping and no compact row, so the whole grouping
machinery of the driver is checked by its result.  Draws are Gumbel-max on Philox4x32-10 at the joint row id (``P.gumbel_scores``).
Wherever the draw is clear the device must have drawn the reference's action; at a near-tie (a top-2 gap within the
heads' error bound: 1e-4 for the exact networks, the replay tolerance for the LSTM) the device's action must be one of the
tied actions and the reference continues with it.  A greedy agent draws nothing but its stuck steps, which are exact: its
actions must always be the reference's."""
import copy

import numpy as np
import torch
import torch.nn.functional as F

import policy_reference as P
from episode_reference import EpisodeReference, rewards_f32
from greedy_reference import GreedyReference
from oracle import cpu
from overcooked_ai_b200.greedy import GreedyHumanModel
from overcooked_ai_b200.selfplay import (PAIR_SALT, PARTNER_DRAW_SALT, PARTNER_MEMBER_SALT, PARTNER_SEAT_SALT, BCPolicy,
                                         RllibLSTMShapedCNN)
from ppo_reference import gae_f32, log_softmax_at

PHI_GAMMA = 0.99        # the potential's gamma of use_phi (the reference's get_state_transition(display_phi=True))
TIE = 1e-4              # libm's log and the device's logf differ in the last bits: a top-2 gap below this may flip
REPLAY_TOL = 0.015      # LSTM heads: |kernel - float64| / (1 + |float64|), bf16 activations at every layer and bf16 h
N_ACTIONS = 6


# ------------------------------------------------------------------------------------------------ per-episode draws
def _env_words(n, key, step):
    """Philox4x32-10 at counter (env lo, env hi, step lo, step hi) for every environment: the per-episode draws' words."""
    e = np.arange(n, dtype=np.uint64)
    ctr = np.stack([e & np.uint64(0xFFFFFFFF), e >> np.uint64(32), np.full_like(e, step & 0xFFFFFFFF),
                    np.full_like(e, step >> 32)], 1).astype(np.uint32)
    return P.philox4x32_10(key, ctr)


def seats_reference(n, seed, step, bc_factor, old, done=None):
    """ovc_assign_partners: paired with probability float32(bc_factor) (word 0 below floor(f 2^32), always at f >= 1), in
    seat word 1 >> 31; -1 = self-play.  done None: every environment, else only where done."""
    w = _env_words(n, seed, step)
    f = float(np.float32(bc_factor))
    thr = 0xFFFFFFFF if f >= 1 else int(f * 4294967296.0) if f > 0 else 0
    hit = (w[:, 0].astype(np.int64) < thr) | (thr == 0xFFFFFFFF)
    new = np.where(hit, (w[:, 1] >> np.uint32(31)).astype(np.int32), -1).astype(np.int32)
    return new if done is None else np.where(done != 0, new, old).astype(np.int32)


def thresholds_reference(weights):
    """The draw table of ovc_assign_members / ovc_assign_pairs: entry k = floor(cdf[k] 2^32), cdf the float64 share of
    entries 0..k (restated here, not imported)."""
    w = np.asarray(weights, np.float64).ravel()
    c = np.cumsum(w)
    return np.floor(c[:-1] / c[-1] * 2.0 ** 32).astype(np.int64)


def members_reference(n, seed, step, thresholds, old, done=None):
    """ovc_assign_members' draw: member = the number of thresholds at or below word 0."""
    w0 = _env_words(n, seed, step)[:, 0].astype(np.int64)
    new = (w0[:, None] >= np.asarray(thresholds, np.int64)[None, :]).sum(1).astype(np.int32)
    return new if done is None else np.where(done != 0, new, old).astype(np.int32)


def pairs_reference(n, K, seed, step, thresholds, old, done=None):
    """ovc_assign_pairs' draw: the ordered pair p = (p // K on player 0, p % K on player 1)."""
    w0 = _env_words(n, seed, step)[:, 0].astype(np.int64)
    p = (w0[:, None] >= np.asarray(thresholds, np.int64)[None, :]).sum(1)
    new = np.stack([p // K, p % K], 1).astype(np.int32)
    return new if done is None else np.where(done[:, None] != 0, new, old).astype(np.int32)


def learner_rows_reference(seat):
    """ovc_learner_rows: (list entries env << 2 | view mask, first compact row, joint rows, row count) of the learner's rows."""
    mask = np.where(seat < 0, 3, np.where(seat == 0, 2, 1)).astype(np.int32)
    cnt = np.where(mask == 3, 2, 1)
    first = (np.cumsum(cnt) - cnt).astype(np.int32)
    jrow = [2 * e + v for e in range(len(seat)) for v in (0, 1) if mask[e] >> v & 1]
    lst = (np.arange(len(seat), dtype=np.int64) << 2 | mask).astype(np.int32)
    return lst, first, np.asarray(jrow, np.int32), int(cnt.sum())


def learner_mask(partner_seat):
    """uint8 [2N]: ``SampleBatch.learner_mask`` of one transition, the rows the learner acts on: both rows of a self-play
    environment (seat -1), the row that is not the partner's otherwise."""
    m = np.ones((len(partner_seat), 2), np.uint8)
    on = partner_seat >= 0
    m[np.flatnonzero(on), partner_seat[on]] = 0
    return m.reshape(-1)


# ------------------------------------------------------------------------------------------------ BC network
def features(tables, lut, states):
    """featurize_state of the oracle, float64 [N, 2, 96] (lut: the layouts' feature LUTs, uint8 [n_layouts, bytes])."""
    return cpu.featurize(tables, lut, states, num_pots=2)


def bc_heads(feats, ops):
    """bf16(features) -> the BC MLP with K8's roundings (ReLU, no input activation); asserts the exactness premise.  K10
    stages the features in bfloat16 (DESIGN §4, K10 "Exactness"): features above 256 (a cook time remaining) are rounded to
    nearest even there, and so they are here."""
    w1, b1, wh, bh, wo, bo = ops
    s, certs = P.k8_reference(P.bf16(feats), w1, b1, wh, bh, wo, bo, 1.0, 0.0)
    assert all(c.holds() for c in certs), "premise: the operands are not exact in float32"
    return s


def bc_operands(bc):
    """A BCPolicy's layers as the float64 operands of ``bc_heads``: heads padded to 8 rows with zeros."""
    d = [(l.weight.detach().double().cpu().numpy(), l.bias.detach().double().cpu().numpy()) for l in bc.dense]
    wo, bo = np.zeros((8, 64)), np.zeros(8)
    n = bc.logits.out_features
    wo[:n], bo[:n] = bc.logits.weight.detach().double().cpu().numpy(), bc.logits.bias.detach().double().cpu().numpy()
    wh = np.stack([w for w, _ in d[1:]]) if len(d) > 1 else np.zeros((0, 64, 64))
    bh = np.stack([b for _, b in d[1:]]) if len(d) > 1 else np.zeros((0, 64))
    return d[0][0], d[0][1], wh, bh, wo, bo


# ------------------------------------------------------------------------------------------------ GAE
def gae_view_f32(rewards, values, dones, last_values, gamma, lam):
    """ovc_gae_view: ``gae_f32`` on one row per environment ([T, N], [T, N], [T, N], [N])."""
    dup = lambda a: np.repeat(np.asarray(a, np.float32), 2, axis=-1)
    adv, tgt = gae_f32(dup(rewards), dup(values), dones, dup(last_values), gamma, lam)
    return adv[:, ::2], tgt[:, ::2]


# ------------------------------------------------------------------------------------------------ CNN premise
def cnn_certificates(cnn, obs):
    """Certificates of every accumulation of ``cnn`` (float64 copy) on observations [M, 2, W, H, 26]: the convolutions as
    matrices over their unfolded inputs, the dense layers and the heads, each on its float64 input; and the largest count of
    significant bits of any operand (activation or weight).  All certificates holding with operands of at most 8 bits
    means every path (bf16 operands, TF32 or float32 GEMMs, any summation order) computes the float64 network."""
    m = copy.deepcopy(cnn).double().cpu().eval()
    x = torch.as_tensor(np.asarray(obs), dtype=torch.float64).reshape(-1, *obs.shape[-3:]).permute(0, 3, 1, 2)
    certs, bits = [], 0
    with torch.no_grad():
        for conv in (m.conv_initial, m.conv_0, m.conv_1):
            k, pad = conv.kernel_size, conv.padding
            cols = F.unfold(x, k, padding=pad).transpose(1, 2).reshape(-1, conv.in_channels * k[0] * k[1])
            w = conv.weight.reshape(conv.out_channels, -1)
            certs.append(P.Certificate(cols.numpy(), w.numpy(), conv.bias.numpy()))
            bits = max(bits, int(P.significant_bits(cols.numpy()).max()), int(P.significant_bits(w.numpy()).max()))
            x = F.leaky_relu(conv(x), 0.2)
        x = x.flatten(1)
        for d in m.dense:
            certs.append(P.Certificate(x.numpy(), d.weight.numpy(), d.bias.numpy()))
            bits = max(bits, int(P.significant_bits(x.numpy()).max()), int(P.significant_bits(d.weight.numpy()).max()))
            x = F.leaky_relu(d(x), m.dense_slope)
        for head in (m.logits, m.value):
            certs.append(P.Certificate(x.numpy(), head.weight.numpy(), head.bias.numpy()))
            bits = max(bits, int(P.significant_bits(head.weight.numpy()).max()))
    return certs, bits


# ------------------------------------------------------------------------------------------------ the agents
class _Agent(object):
    """One policy as the reference evaluates it: ``kind`` cnn / lstm / bc / greedy, its draw key and the name of its
    counter."""

    def __init__(self, model, key, counter, host):
        self.model, self.key, self.counter = model, int(key) & (2**64 - 1), counter
        self.kind = "bc" if isinstance(model, BCPolicy) else "lstm" if isinstance(model, RllibLSTMShapedCNN) else \
            "greedy" if isinstance(model, GreedyHumanModel) else "cnn"
        self.host = host
        self.h = self.c = None  # LSTM: float64 state per joint row [2N, cell]
        self.greedy = None      # greedy: its GreedyReference (previous states per environment)
        self.sync()

    def sync(self):
        """Take the model's current weights (``sync_weights``)."""
        if self.kind == "greedy":
            if self.greedy is None:  # salted inside GreedyReference, as the device passes seed ^ GREEDY_DRAW_SALT
                self.greedy = GreedyReference(self.host.layouts, self.key, self.host.n)
            return
        if self.kind == "bc":
            self.ops = bc_operands(self.model)
        else:
            self.m64 = copy.deepcopy(self.model).double().cpu().eval()
        if self.kind == "lstm" and self.h is None:
            cell = self.model.lstm.hidden_size
            self.h, self.c = np.zeros((2 * self.host.n, cell)), np.zeros((2 * self.host.n, cell))

    def greedy_actions(self, state, rows, done, step):
        """The greedy agent's actions on joint rows ``rows``: ``GreedyReference.act`` on every environment, with the player
        it holds there (-1 where it holds none, which forgets the previous state), the previous transition's episode ends
        and its draw counter ``step``."""
        player = np.full(self.host.n, -1, np.int64)
        player[rows // 2] = rows % 2
        self.greedy.step = step
        return self.greedy.act(state, player, done)[rows // 2]

    def heads(self, cache, rows, reset):
        """(scores [len(rows), 8] with the value in column 6, values [len(rows)]) of this agent on joint rows ``rows``; an
        LSTM advances its state on those rows, zeroed first where ``reset`` (per joint row)."""
        if len(rows) == 0:
            return np.zeros((0, 8)), np.zeros(0)
        if self.kind == "bc":
            s = bc_heads(cache.feats()[rows], self.ops)
            return s, np.full(len(rows), np.nan)
        x = cache.obs64()[torch.as_tensor(rows)]
        with torch.no_grad():
            if self.kind == "cnn":
                lg, v = self.m64(x)
            else:
                keep = torch.as_tensor(~reset[rows]).unsqueeze(1)
                h = torch.where(keep, torch.as_tensor(self.h[rows]), torch.zeros(1, dtype=torch.float64))
                c = torch.where(keep, torch.as_tensor(self.c[rows]), torch.zeros(1, dtype=torch.float64))
                lg, v, (h, c) = self.m64(x, (h, c))
                self.h[rows], self.c[rows] = h.numpy(), c.numpy()
        s = np.zeros((len(rows), 8))
        s[:, :N_ACTIONS], s[:, N_ACTIONS] = lg.numpy(), v.numpy()
        return s, v.numpy()


class _StateCache(object):
    """The observation and the features of one state, computed on first use."""

    def __init__(self, host, state):
        self.host, self.state, self._obs, self._feats = host, state, None, None

    def obs64(self):
        if self._obs is None:
            h = self.host
            o = cpu.encode_lossless(h.tables, self.state, h.W, h.H, h.horizon)
            self._obs = torch.as_tensor(o, dtype=torch.float64).reshape(-1, h.W, h.H, 26).permute(0, 3, 1, 2)
        return self._obs

    def feats(self):
        if self._feats is None:
            self._feats = features(self.host.tables, self.host.lut, self.state).reshape(2 * self.host.n, -1)
        return self._feats


class EnvHost(object):
    """What the reference needs of the environments, as host arrays: layout tables and start records, the horizon, the
    random-start parameters (``cpu.random_start`` or None), the grid, the feature LUTs, the 0.99 potential tables (pt, cost
    LUT, gamma powers), each layout's delivery values, the environment count, and the compiled layouts (the greedy
    agent's planners)."""

    def __init__(self, tables, starts, horizon, rs, W, H, lut, pot, deliver_value, n, layouts=None):
        self.tables, self.starts, self.horizon, self.rs = tables, starts, horizon, rs
        self.W, self.H, self.lut, self.pot, self.deliver_value, self.n = W, H, lut, pot, deliver_value, n
        self.layouts = layouts


# ------------------------------------------------------------------------------------------------ the rollout
class RolloutReference(object):
    """A rollout restated.  ``spec`` (a dict) describes it:

    kind          "self_play" or "pair"
    learner       self_play: a model or a list of models (a population of learners)
    blocks        environment counts per member (blocks; default equal) when ``learner`` is a list without pairs
    pairs / pair_weights   population play: int32 [N, 2] fixed pairs, or K x K weights drawn per episode
    partner       self_play: None, a BCPolicy, a GreedyHumanModel, an RllibShapedCNN, or a list of members (a population)
    member / member_weights   a population of partners (self_play) or agent 1's population (pair): fixed int32 [N] or drawn
    bc_factor     the seat draw's factor (self_play with a partner)
    agents        pair: (agent0, agent1 or a list of members)
    swap          pair: int32 [N] or None;  random_seats: pair, the seats drawn per episode
    seed, factor (reward_shaping_factor), use_phi, capacity (episode_capacity), seq_len (max_seq_len)

    ``state`` is the environments' records at construction.  A collect() window with ``bootstrap_horizon``
    (``begin_window``) also returns each transition's ``terminal_values``."""

    def __init__(self, host, state, spec):
        self.host, self.spec = host, dict(spec)
        n = self.n = host.n
        self.state = np.array(state, np.int32)
        self.seed = int(spec.get("seed", 0))
        self.factor = float(spec.get("factor", 1.0))
        self.use_phi = bool(spec.get("use_phi", False))
        self.seq_len = int(spec.get("seq_len", 20))
        self.pair_kind = spec["kind"] == "pair"
        self.counters = {}
        self.prev_done = np.zeros(n, bool)
        self.ret_sparse = np.zeros(n, np.int64)
        self.ret_mixed = np.zeros(n, np.float32)
        lid = self.state[:, 3] & 0xFF
        self.ep = EpisodeReference(host.deliver_value, lid, int(spec.get("capacity", 1)), members=self._has_members(),
                                   pairs=self._has_pairs())
        self.run_records = self.ep.save_records()
        self.partner_seat = np.full(n, -1, np.int32)
        self.member = self.pair = None
        self.member_thr = self.pair_thr = None
        self.bc = float(spec.get("bc_factor", 0.0))
        self.ties = self.draws = 0        # near-ties of the exact networks' draws, and all their draws
        self.lstm_open = self.lstm_draws = 0  # LSTM draws within the heads' error bound (checked only as one of the tied), all
        self.bootstrap_horizon = False    # the current window's collect(bootstrap_horizon=...)
        self.terminal_records = []        # the terminal records the window's terminal values were evaluated on
        if self.pair_kind:
            self._init_pair(spec)
        else:
            self._init_self_play(spec)

    # -------------------------------------------------------------------- construction
    def _has_members(self):
        s = self.spec
        return isinstance(s.get("partner"), (list, tuple)) or (self.pair_kind and isinstance(s["agents"][1], (list, tuple)))

    def _has_pairs(self):
        return self.spec.get("pairs") is not None or self.spec.get("pair_weights") is not None

    def _count(self, name):
        self.counters.setdefault(name, 0)
        return name

    def _init_population(self, members, member, weights, key_base):
        """Member agents (each its own counter) and the member table: fixed, or drawn at construction."""
        self.members = [_Agent(m, self.seed ^ PARTNER_DRAW_SALT if isinstance(m, BCPolicy) else self.seed,
                               self._count("%s%d" % (key_base, k)), self.host) for k, m in enumerate(members)]
        if member is not None:
            self.member = np.array(member, np.int32)
        else:
            self.member_weights = [1.0] * len(members) if weights is None else list(weights)
            self.member_thr = thresholds_reference(self.member_weights)
            self._count("member_draw")
            self.member = members_reference(self.n, self.seed ^ PARTNER_MEMBER_SALT, self._advance("member_draw"), self.member_thr, None)

    def _advance(self, name):
        v = self.counters[name]
        self.counters[name] = v + 1
        return v

    def _init_self_play(self, s):
        n = self.n
        learners = list(s["learner"]) if isinstance(s["learner"], (list, tuple)) else [s["learner"]]
        self.learners = [_Agent(m, self.seed, self._count("draw"), self.host) for m in learners]
        K = len(learners)
        self.block_member = None
        if self._has_pairs():
            if s.get("pairs") is not None:
                self.pair = np.array(s["pairs"], np.int32)
            else:
                self.pair_weights = np.asarray(s["pair_weights"], np.float64)
                self.pair_thr = thresholds_reference(self.pair_weights)
                self._count("pair_draw")
                self.pair = pairs_reference(n, K, self.seed ^ PAIR_SALT, self._advance("pair_draw"), self.pair_thr, None)
        elif K > 1:
            counts = s.get("blocks") or [(k + 1) * n // K - k * n // K for k in range(K)]
            self.block_member = np.repeat(np.arange(K), counts).astype(np.int32)
        p = s.get("partner")
        self.partner = None
        if p is not None:
            if isinstance(p, (BCPolicy, GreedyHumanModel)):
                key = self.seed ^ PARTNER_DRAW_SALT if isinstance(p, BCPolicy) else self.seed
                self.partner = _Agent(p, key, self._count("partner"), self.host)
            else:
                members = list(p) if isinstance(p, (list, tuple)) else [p]
                member = np.zeros(n, np.int32) if not isinstance(p, (list, tuple)) else s.get("member")
                self._init_population(members, member, s.get("member_weights"), "member")
                self.partner = "population"
            self._count("seat")
            self.partner_seat = seats_reference(n, self.seed ^ PARTNER_SEAT_SALT, self._advance("seat"), self.bc, None)

    def _init_pair(self, s):
        n = self.n
        a0, a1 = s["agents"]
        self.random_seats = bool(s.get("random_seats", False))
        if self.random_seats:
            self._count("seat")
            self.partner_seat = seats_reference(n, self.seed ^ PARTNER_SEAT_SALT, self._advance("seat"), 1.0, None)
        else:
            swap = s.get("swap")
            self.partner_seat = np.ones(n, np.int32) if swap is None else (1 ^ (np.asarray(swap) != 0)).astype(np.int32)
        key = lambda m: self.seed ^ PARTNER_DRAW_SALT if isinstance(m, BCPolicy) else self.seed
        self.agent0 = _Agent(a0, key(a0), self._count("agent0"), self.host)
        if isinstance(a1, (list, tuple)):
            self._init_population(list(a1), s.get("member"), s.get("member_weights"), "member")
            self.agent1 = "population"
        else:
            self.agent1 = _Agent(a1, key(a1), self._count("agent1"), self.host)

    # -------------------------------------------------------------------- setters between windows
    def set_member_weights(self, w):
        self.member_weights = list(w)
        self.member_thr = thresholds_reference(w)

    def set_pair_weights(self, w):
        self.pair_weights = np.asarray(w, np.float64)
        self.pair_thr = thresholds_reference(self.pair_weights)

    def sync(self):
        for a in self.agents():
            a.sync()

    def agents(self):
        out = [self.agent0] if self.pair_kind else list(self.learners)
        other = self.agent1 if self.pair_kind else self.partner
        if other == "population":
            out += self.members
        elif other is not None:
            out.append(other)
        return out

    # -------------------------------------------------------------------- rows
    def _learner_of_row(self):
        """int [2N]: the learner member that holds each joint row as if no partner played (self-play, blocks or pairs)."""
        n = self.n
        if self.pair is not None:
            return self.pair.reshape(-1).copy()
        if self.block_member is not None:
            return np.repeat(self.block_member, 2)
        return np.zeros(2 * n, np.int64)

    def holders(self):
        """[(agent, joint rows)] of this transition: every row's agent, each evaluated on its own rows only."""
        n, e = self.n, np.arange(self.n)
        ps = self.partner_seat
        paired = ps >= 0
        prow = 2 * e[paired] + ps[paired]   # the partner's (agent 1's) rows
        out = []
        if self.pair_kind:
            out.append((self.agent0, 2 * e + (1 - ps)))
        else:
            lrow = np.setdiff1d(np.arange(2 * n), prow)
            who = self._learner_of_row()[lrow]
            out += [(a, lrow[who == k]) for k, a in enumerate(self.learners)]
        other = self.agent1 if self.pair_kind else self.partner
        if other == "population":
            mem = self.member[e[paired]]
            out += [(a, prow[mem == k]) for k, a in enumerate(self.members)]
        elif other is not None:
            out.append((other, prow))
        return out

    # -------------------------------------------------------------------- the draw
    def _draw(self, scores, rows, key, step, known, lstm):
        """The actions of ``rows`` (Gumbel-max at the joint row, ``key``, ``step``), checked against the device's ``known``
        actions (-1: not known) where the draw is clear; near-ties keep the device's action, or stay open (a list of the
        tied actions) where it is not known."""
        if len(rows) == 0:
            return np.zeros(0, np.int64), {}
        v = P.gumbel_scores(scores, key, step, N_ACTIONS, rows)
        top = v.max(1)
        bound = np.full((len(rows), 1), TIE)
        if lstm:
            bound = np.maximum(bound, 2 * REPLAY_TOL * (1 + np.abs(scores[:, :N_ACTIONS]).max(1, keepdims=True)))
        tied = v >= top[:, None] - bound
        want = v.argmax(1)
        k = known[rows]
        loose = np.flatnonzero(tied.sum(1) > 1)
        if lstm:
            self.lstm_draws += len(rows)
            self.lstm_open += len(loose)
        else:
            self.draws += len(rows)
            self.ties += len(loose)
        open_ = {}
        for i in loose:
            if k[i] >= 0:
                assert tied[i, k[i]], ("device action %d is not among the tied actions %s at row %d"
                                       % (k[i], np.flatnonzero(tied[i]).tolist(), rows[i]))
                want[i] = k[i]
            else:
                open_[int(rows[i])] = np.flatnonzero(tied[i]).tolist()
        clear = tied.sum(1) == 1
        bad = clear & (k >= 0) & (k != want)
        assert not bad.any(), "draw differs at joint rows %s: device %s, reference %s" % (
            rows[bad][:8].tolist(), k[bad][:8].tolist(), want[bad][:8].tolist())
        return want, open_

    # -------------------------------------------------------------------- one transition
    def transition(self, known=None, next_state=None, next_reward=None):
        """One transition from ``self.state``.  ``known``: the device's joint actions int [2N] (-1 where not known), used
        at near-ties and checked wherever the draw is clear; ``next_state`` and ``next_reward`` (player [N], reward [N]): the
        device's records after the transition and one player's reward, which settle a near-tie on a row whose action is not
        known.  Returns the transition's outputs as a dict."""
        n, host = self.n, self.host
        known = np.full(2 * n, -1, np.int64) if known is None else np.asarray(known, np.int64)
        cache = _StateCache(host, self.state)
        out = {"state": self.state.copy(), "partner_seat": self.partner_seat.copy(),
               "member": None if self.member is None else self.member.copy(), "pair": None if self.pair is None else self.pair.copy()}
        scores, values = np.full((2 * n, 8), np.nan), np.full(2 * n, np.nan)
        actions = np.full(2 * n, -1, np.int64)
        reset = np.repeat(self.prev_done, 2)
        open_rows = {}
        steps = {}
        for agent, rows in self.holders():
            if agent.counter not in steps:  # learner members share one counter: one advance per transition
                steps[agent.counter] = self._advance(agent.counter)
            if agent.kind == "greedy":  # no Gumbel draw and no tie: every known action must be the reference's
                a = agent.greedy_actions(self.state, rows, self.prev_done, steps[agent.counter])
                k = known[rows]
                bad = (k >= 0) & (k != a)
                assert not bad.any(), "greedy action differs at joint rows %s: device %s, reference %s" % (
                    rows[bad][:8].tolist(), k[bad][:8].tolist(), a[bad][:8].tolist())
                actions[rows] = a
                continue
            s, v = agent.heads(cache, rows, reset)
            scores[rows], values[rows] = s, v
            a, op = self._draw(s, rows, agent.key, steps[agent.counter], known, agent.kind == "lstm")
            actions[rows] = a
            open_rows.update(op)
        lstm = None if self.pair_kind else self.lstm_agent()
        if lstm is not None:  # the LSTM learner runs on all 2N rows (K11 has no rows form): the partner's rows' state too
            lstm.heads(cache, np.setdiff1d(np.arange(2 * n), np.concatenate([r for a, r in self.holders() if a is lstm])), reset)
        for agent in self.agents():  # an agent with no rows this transition still advances its counter once
            if agent.counter not in steps:
                steps[agent.counter] = self._advance(agent.counter)
        if open_rows:
            self._settle(actions, open_rows, next_state, next_reward)
        joint = actions.reshape(n, 2).astype(np.int32)
        sparse, shaped, done, events, nxt, rewards, dense, term = self._step(self.state, joint, self.bootstrap_horizon)
        if self.bootstrap_horizon:
            out["terminal_values"] = self._terminal_values(term, done != 0, reset)
        self.state = nxt
        f = np.float32(self.factor)
        if dense is None:
            sh = shaped.astype(np.float32)
            self.ret_mixed = (((self.ret_mixed + sparse.astype(np.float32)) + f * sh[:, 0]) + f * sh[:, 1]).astype(np.float32)
        else:
            self.ret_mixed = (((self.ret_mixed + sparse.astype(np.float32)) + f * dense) + f * dense).astype(np.float32)
        self.ret_sparse += sparse
        d = done != 0
        # the member and pair draws run after K1 and before the record: the ending episode's member / pair is recorded
        rec_member = None if self.member is None else self.member.copy()
        rec_pair = None if self.pair is None else self.pair.copy()
        if self.member_thr is not None:
            self.member = members_reference(n, self.seed ^ PARTNER_MEMBER_SALT, self._advance("member_draw"), self.member_thr,
                                            self.member, done)
        if self.pair_thr is not None:
            self.pair = pairs_reference(n, len(self.learners), self.seed ^ PAIR_SALT, self._advance("pair_draw"), self.pair_thr,
                                        self.pair, done)
        has_seat = self.pair_kind or self.partner is not None
        self.ep.step(shaped, done, events, self.state[:, 3] & 0xFF, rewards, self.partner_seat if has_seat else None,
                     member=rec_member, pair=rec_pair)
        # the seat draw runs after the record: the ending episode's seats went into it
        if "seat" in self.counters:
            bc = 1.0 if self.pair_kind else self.bc
            self.partner_seat = seats_reference(n, self.seed ^ PARTNER_SEAT_SALT, self._advance("seat"), bc, self.partner_seat, done)
        self.prev_done = d
        out.update(actions=actions, scores=scores, values=values, rewards=rewards, dones=d.astype(np.uint8),
                   logp=self._logp(scores, actions))
        return out

    def _step(self, state, joint, terminal=False):
        """K1 with its auto-reset from ``state`` (not modified), and the rewards: ``sparse + factor * shaped_i``, or with
        use_phi ``sparse + factor * float32(phi(s') - phi(s))``, s' taken before the reset.  Returns (sparse, shaped, done,
        events, the next records, rewards [N, 2], the dense reward or None, the records of K1 without the reset (the
        ended episodes' terminal records) with use_phi or ``terminal``, else None)."""
        h = self.host
        nxt = state.copy()
        sparse, shaped, done, events = cpu.step(h.tables, h.starts, nxt, joint, horizon=h.horizon, flags=1, rs=h.rs)
        f = np.float32(self.factor)
        term = None
        if self.use_phi or terminal:
            term = state.copy()
            cpu.step(h.tables, h.starts, term, joint, horizon=h.horizon, flags=0, rs=h.rs)
        if not self.use_phi:
            return sparse, shaped, done, events, nxt, rewards_f32(sparse, shaped, self.factor), None, term
        pt, cl, gpow = h.pot
        dense = (cpu.potential(h.tables, pt, cl, gpow, term) - cpu.potential(h.tables, pt, cl, gpow, state)).astype(np.float32)
        r = (sparse.astype(np.float32) + f * dense).astype(np.float32)
        return sparse, shaped, done, events, nxt, np.stack([r, r], 1), dense, term

    def _terminal_values(self, term, d, reset):
        """float32 [2N]: the horizon bootstrap's value pass, the learner's float64 value on the terminal records ``term``
        at its rows of the environments that ended (``d``) — both rows in self-play, row 1 - partner_seat when paired, agent
        0's row of a pair — and 0 on every other row."""
        n = self.n
        if self.pair_kind:
            learner, mine = self.agent0, np.zeros(2 * n, bool)
            mine[2 * np.arange(n) + (1 - self.partner_seat)] = True
        else:
            learner, mine = self.learners[0], learner_mask(self.partner_seat).astype(bool)
        rows = np.flatnonzero(np.repeat(d, 2) & mine)
        out = np.zeros(2 * n, np.float32)
        out[rows] = learner.heads(_StateCache(self.host, term), rows, reset)[1]
        self.terminal_records.append(term[d])
        return out

    def _settle(self, actions, open_rows, next_state, next_reward):
        """Near-ties on rows whose device action is not known: the tied action whose oracle step gives the device's next
        records of that environment and, where ``next_reward`` = (player [N], reward [N]) is given, the device's reward of
        that player (an episode's last action is hidden by the reset, not by the reward); any, where they cannot tell."""
        assert next_state is not None, "a near-tie on a row whose device action is unknown, and no next state to settle it"
        h = self.host
        for e in sorted({r // 2 for r in open_rows}):
            opts = [[a] for a in open_rows.get(2 * e, [actions[2 * e]])]
            opts = [(a, b) for (a,) in opts for b in open_rows.get(2 * e + 1, [actions[2 * e + 1]])]
            fit = []
            for a, b in opts:  # the whole batch: a random reset draws from the environment's index
                joint = np.maximum(actions, 0).reshape(-1, 2).astype(np.int32)
                joint[e] = a, b
                _, _, _, _, s, r, _, _ = self._step(self.state, joint)
                if np.array_equal(s[e], next_state[e]) and (next_reward is None or r[e, next_reward[0][e]] == next_reward[1][e]):
                    fit.append((a, b))
            assert fit, "no tied action reaches the device's next state in environment %d" % e
            actions[2 * e], actions[2 * e + 1] = fit[0]

    @staticmethod
    def _logp(scores, actions):
        lp = np.full(len(actions), np.nan)
        ok = ~np.isnan(scores[:, 0])
        lp[ok] = log_softmax_at(scores[ok], actions[ok], N_ACTIONS)
        return lp

    # -------------------------------------------------------------------- learner-side views

    def bootstrap(self):
        """The learner's values on the state after a window: self-play, every joint row by its learner member (the partner's
        rows too); a pair, agent 0's row of each environment [N].  Draws nothing the rollout keeps, so it advances no counter
        and leaves the LSTM state alone."""
        n = self.n
        cache = _StateCache(self.host, self.state)
        reset = np.repeat(self.prev_done, 2)
        if self.pair_kind:
            rows = 2 * np.arange(n) + (1 - self.partner_seat)
            agents = [(self.agent0, rows)]
        else:
            who = self._learner_of_row()
            agents = [(a, np.flatnonzero(who == k)) for k, a in enumerate(self.learners)]
        vals = np.full(2 * n, np.nan)
        for a, rows in agents:
            saved = None if a.kind != "lstm" else (a.h.copy(), a.c.copy())
            vals[rows] = a.heads(cache, rows, reset)[1]
            if saved is not None:
                a.h, a.c = saved
        return vals[2 * np.arange(n) + (1 - self.partner_seat)] if self.pair_kind else vals

    def lstm_agent(self):
        """The learner's LSTM agent (self-play learner or pair agent 0), or None."""
        a = self.agent0 if self.pair_kind else self.learners[0]
        return a if a.kind == "lstm" else None

    # -------------------------------------------------------------------- windows
    def begin_window(self, n_steps, bootstrap_horizon=False):
        """collect()'s records: a batch holds ceil(T / horizon) episodes per environment, the most T transitions can end;
        with ``bootstrap_horizon`` each transition also returns the terminal values."""
        self.ep.load_records(self.ep.empty_records(-(-int(n_steps) // self.host.horizon)))
        self.bootstrap_horizon, self.terminal_records = bool(bootstrap_horizon), []

    def end_window(self):
        self.bootstrap_horizon = False
        return self.ep.save_records()

    def begin_run(self):
        self.ep.load_records(self.run_records)

    def end_run(self):
        self.run_records = self.ep.save_records()
