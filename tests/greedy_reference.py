"""A host restatement of the reference's ``GreedyHumanModel.action`` (agents/agent.py) with its defaults (no Boltzmann
options, ``auto_unstuck=True``) on packed records, in numpy, for the tests of the greedy kernel.

It follows the reference's steps rather than the kernel's tables: ``ml_action`` builds the goal list from feature
positions (``MediumLevelActionManager``'s pickup / pot / soup / serve actions, counter objects included), filters it with
``MotionPlanner.is_valid_motion_start_goal_pair`` (a goal faces a non-floor cell that is not a counter — NO_COUNTERS_PARAMS
has no counter goals — and lies in the start's connected component), falls back to ``go_to_closest_feature_actions``
and takes the first cheapest goal of the list (``get_lowest_cost_action_and_goal``'s strict ``<``).  The plans
themselves are ``greedy.plan_table``'s, which tests/test_greedy_cpu.py checks against a BFS of the motion graph.

Deliberate differences from the reference, which the kernel shares: a stuck step draws its action with Philox4x32-10
(``stuck_draw``) instead of numpy, and objects on counters are listed in record slot order instead of
``state.objects`` insertion order (those goals are refused by the valid-goal filter either way).
"""
import numpy as np

from overcooked_ai_b200 import greedy as G
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.actions import Direction

GREEDY_DRAW_SALT = G.GREEDY_DRAW_SALT


def philox4x32_10(key, c0, c1, c2, c3):
    k0, k1 = key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c3 ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def stuck_draw(seed, row, step, n):
    """The index of a stuck step's action in its unblocking set of n actions: word 0 of Philox4x32-10 with key ``seed ^
    GREEDY_DRAW_SALT``, counter (row lo, row hi, step lo, step hi) on the joint row 2 e + p, scaled by multiply-high."""
    v = philox4x32_10((seed ^ GREEDY_DRAW_SALT) & (2**64 - 1), row & 0xFFFFFFFF, row >> 32, step & 0xFFFFFFFF, step >> 32)
    return (v[0] * n) >> 32


class LayoutPlanner(object):
    """One layout's motion planner: node numbering, motion goals and plans (``greedy.plan_table``)."""

    def __init__(self, cl):
        G.check_layout(cl)
        self.cl = cl
        self.free = list(cl.terrain_pos_dict[" "])
        self.index = {p: i for i, p in enumerate(self.free)}
        self.plan = G.plan_table(cl)

    def node(self, word):
        w = int(word) & 0xFFFFFFFF
        return 4 * self.index[L.byte_pos(w & 0xFF)] + ((w >> 8) & 3)

    def is_valid_goal(self, start, goal):
        i, o = divmod(goal, 4)
        d = Direction.INDEX_TO_DIRECTION[o]
        p = self.free[i]
        facing = self.cl.get_terrain_type_at_pos((p[0] + d[0], p[1] + d[1]))
        if facing in (" ", "X"):  # NO_COUNTERS_PARAMS: counter_goals = []
            return False
        return self.plan[start, goal] != G.PLAN_UNREACHABLE

    def goals_for(self, positions):
        return [g for p in positions for g in G.motion_goals(self.cl, p)]


def pot_states(cl, rec):
    """``get_pot_states`` (overcooked_mdp.py): {'empty', 'ready', 'cooking', '<n>_items'} -> pot positions, pot order."""
    out = {}
    for k, pos in enumerate(cl.pot_locations):
        code = int(rec[4 + k]) & L.OBJ_MASK
        if code & 7 == L.O_NONE:
            key = "empty"
        else:
            n = (code >> 3) & 3
            n_tom = bin((code >> 5) & ((1 << n) - 1)).count("1")
            tick = ((code >> 8) & 0x3FFF) - 1
            cook = int(cl.cook_time[(n - n_tom) * 4 + n_tom])
            key = "%d_items" % n if tick < 0 else ("ready" if tick >= cook else "cooking")
        out.setdefault(key, []).append(pos)
    return out


def partially_full(ps):
    """get_partially_full_pots: list(set().union(one_item_pots, two_item_pots)), CPython's set order."""
    return list(set().union(*[ps.get("1_items", []), ps.get("2_items", [])]))


def counter_objects(cl, rec):
    """get_counter_objects_dict over every counter: name -> positions (record slot order)."""
    out = {}
    for k in range(cl.n_pots, cl.n_slots):
        t = int(rec[4 + k]) & 7
        if t:
            out.setdefault(L.OBJ_NAME[t], []).append(cl.slot_positions[k])
    return out


def ml_action(lp, rec, p):
    """``GreedyHumanModel.ml_action``: the valid motion goals of player p (node numbers, list order)."""
    cl = lp.cl
    me, other = int(rec[1 + p]) & 0xFFFFFFFF, int(rec[2 - p]) & 0xFFFFFFFF
    held, other_held = (me >> 10) & 7, (other >> 10) & 7
    T = cl.terrain_pos_dict
    counters = counter_objects(cl, rec)
    ps = pot_states(cl, rec)
    if held == L.O_NONE:
        nearly_ready = bool(ps.get("ready")) or bool(ps.get("cooking"))
        if nearly_ready and other_held != L.O_DISH:
            positions = T["D"] + counters.get("dish", [])
        elif ps.get("3_items"):  # start_cooking_actions({'3_items': ...}): no partial pots in that dict
            positions = ps["3_items"]
        else:
            positions = T["O"] + counters.get("onion", [])
    elif held in (L.O_ONION, L.O_TOMATO):
        positions = partially_full(ps) + ps.get("empty", [])
    elif held == L.O_DISH:
        positions = ps.get("ready", []) + ps.get("cooking", [])
    else:
        positions = T["S"]
    start = lp.node(me)
    goals = [g for g in lp.goals_for(positions) if lp.is_valid_goal(start, g)]
    if not goals:  # go_to_closest_feature_actions: the first cheapest feature, then its goals
        best, best_f = None, None
        for f in T["O"] + T["T"] + cl.pot_locations + T["D"]:
            for g in G.motion_goals(cl, f):
                if lp.is_valid_goal(start, g) and (best is None or lp.plan[start, g] >> 3 < best):
                    best, best_f = lp.plan[start, g] >> 3, f
        goals = [] if best_f is None else [g for g in G.motion_goals(cl, best_f) if lp.is_valid_goal(start, g)]
    return start, goals


def planned_action(lp, rec, p):
    """The action of ``get_lowest_cost_action_and_goal`` over ml_action's goals (STAY where there is none: the reference
    asserts there is one)."""
    start, goals = ml_action(lp, rec, p)
    best, act = None, G.A_STAY
    for g in goals:
        c = int(lp.plan[start, g]) >> 3
        if best is None or c < best:
            best, act = c, int(lp.plan[start, g]) & 7
    return act


def unblocking_actions(lp, rec, p):
    """auto_unstuck's unblocking set: the moves N, S, E, W (action order) that change player p's position while the other
    player stays, i.e. into a floor cell the other player does not hold."""
    me, other = int(rec[1 + p]) & 0xFF, int(rec[2 - p]) & 0xFF
    pos, opos = L.byte_pos(me), L.byte_pos(other)
    out = []
    for a, d in enumerate(Direction.ALL_DIRECTIONS):
        q = (pos[0] + d[0], pos[1] + d[1])
        if q in lp.index and q != opos:
            out.append(a)
    return out


def players_key(rec):
    """Both players' position and orientation (``state.players_pos_and_or``)."""
    return ((int(rec[1]) & 0x3FF), (int(rec[2]) & 0x3FF))


def state_key(rec):
    """players_key in the kernel's ``prev`` encoding: bits 0-9 / 10-19 players 0 / 1, bit 20 valid."""
    k0, k1 = players_key(rec)
    return k0 | (k1 << 10) | (1 << 20)


class GreedyReference(object):
    """The greedy agent over N environments, step by step: ``act(records, player, done)`` returns its action per
    environment (-1 where player[e] < 0), as the kernel computes it from the same inputs.  ``prev`` holds each
    environment's previous state key in the kernel's encoding (``state_key``; 0: no previous state, as after
    ``Agent.reset()``); ``step`` is the draw counter."""

    def __init__(self, layouts, seed, n_envs):
        self.planners = [LayoutPlanner(cl) for cl in layouts]
        self.seed, self.step = int(seed), 0
        self.prev = [0] * n_envs

    def act(self, records, player, done=None):
        out = np.full(len(records), -1, np.int64)
        for e, rec in enumerate(records):
            p = int(player[e])
            if p < 0 or (done is not None and done[e]):
                self.prev[e] = 0
            if p < 0:
                continue
            lp = self.planners[int(rec[3]) & 0xFF]
            key = state_key(rec)
            act = planned_action(lp, rec, p)
            if self.prev[e] == key:
                unblock = unblocking_actions(lp, rec, p)
                act = unblock[stuck_draw(self.seed, 2 * e + p, self.step, len(unblock))] if unblock else G.A_STAY
            self.prev[e] = key
            out[e] = act
        self.step += 1
        return out
