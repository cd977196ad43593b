"""The reference's scripted partner ``GreedyHumanModel`` (agents/agent.py) on the device: its motion plans as per-layout
tables built once here, its per-step decision in the CUDA kernel of include/ovc_greedy.h.

Under the planner parameters the reference plays it with (``NO_COUNTERS_PARAMS``, planning/planners.py:27-34) a motion
plan depends only on its (start, goal) pair of (floor cell, orientation) states, so ``MotionPlanner``'s whole plan
dictionary becomes one table per layout: for every pair the plan's first action and its cost.  What is left per step is
the choice of the goal set from the pots and the held objects (``ml_action``) and an argmin over table lookups
(``get_lowest_cost_action_and_goal``), which the kernel makes for every environment in one thread.

Node n of a layout's motion graph is ``4 * i + o``: floor cell i in ``terrain_pos_dict[' ']`` order (row-major) facing
orientation o (N, S, E, W), the reference's state-encoder order (``get_valid_player_positions_and_orientations``).
"""
from collections import deque

import numpy as np

from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.actions import Direction

# A stuck step's draw (auto_unstuck) uses key seed ^ GREEDY_DRAW_SALT, so it never reuses the noise of another draw keyed
# by the rollout's seed on the same (env, step) counter.
GREEDY_DRAW_SALT = 0xBF58476D1CE4E5B9
PLAN_UNREACHABLE = 0xFFFF
A_STAY, A_INTERACT = 4, 5
MAX_NODES = 4 * L.MAX_FREE
MAX_GOALS = 1024
# goal lists of the table: onion dispensers, dish dispensers, serving cells, go_to_closest_feature's features, pot k
LIST_ONION, LIST_DISH, LIST_SERVE, LIST_CLOSEST, LIST_POT = 0, 1, 2, 3, 4
N_LISTS = LIST_POT + L.MAX_POTS

GREEDY_LAYOUT_DTYPE = np.dtype(
    [
        ("n_nodes", "<i4"), ("plan_offset", "<i4"),
        ("list_start", "<u2", (N_LISTS + 1,)), ("reserved", "<u2", (3,)),
        ("free_index", "u1", (256,)), ("partial_order", "u1", (81, L.MAX_POTS)),
        ("goal", "<u2", (MAX_GOALS,)),
    ]
)
assert GREEDY_LAYOUT_DTYPE.itemsize == 2660


class GreedyHumanModel(object):
    """The reference's ``GreedyHumanModel(MediumLevelActionManager(mdp, NO_COUNTERS_PARAMS))`` with its defaults, as an
    agent of ``AgentPairRollout`` or the ``partner`` of ``SelfPlayRollout``: it needs no weights.  Only the defaults are
    built: the Boltzmann-rational variants draw goals and motions from softmaxes of plan costs and are refused, and so is
    ``auto_unstuck=False``."""

    def __init__(self, hl_boltzmann_rational=False, ll_boltzmann_rational=False, hl_temp=1, ll_temp=1, auto_unstuck=True):
        if hl_boltzmann_rational or ll_boltzmann_rational or not auto_unstuck:
            raise ValueError("GreedyHumanModel on the device plays the reference's defaults only: no Boltzmann-rational "
                             "goal or motion choice, auto_unstuck=True")

    def __repr__(self):
        return "GreedyHumanModel()"


def check_layout(cl):
    """The orders ``ml_action`` accepts (agent.py: 'only support 3-onion-soup order'): exactly one order, of three onions."""
    orders = cl.start_all_orders
    if len(orders) != 1 or list(orders[0]["ingredients"]) != ["onion"] * 3:
        raise ValueError("GreedyHumanModel plays layouts with one order of three onions (its ml_action asserts it); "
                         "layout %r has orders %r" % (cl.layout_name, orders))


def motion_graph(cl):
    """(free cells, succ int32 [n, 4]): MotionPlanner's graph (planners.py:315-358) — from node (p, o), direction action a
    moves to p + a facing a where that is floor, else turns in place to face a (_move_if_direction); STAY and INTERACT are
    self-loops, which no shortest path uses."""
    free = list(cl.terrain_pos_dict[" "])
    index = {p: i for i, p in enumerate(free)}
    succ = np.zeros((4 * len(free), 4), np.int32)
    for i, p in enumerate(free):
        for o in range(4):
            for a, d in enumerate(Direction.ALL_DIRECTIONS):
                q = (p[0] + d[0], p[1] + d[1])
                succ[4 * i + o, a] = 4 * index[q] + a if q in index else 4 * i + a
    return free, succ


def motion_goals(cl, feature):
    """``motion_goals_for_pos[feature]`` (planners.py:439-450): the nodes next to the feature cell facing it, in N, S, E,
    W order of the side they lie on."""
    free = list(cl.terrain_pos_dict[" "])
    index = {p: i for i, p in enumerate(free)}
    out = []
    for d in Direction.ALL_DIRECTIONS:
        q = (feature[0] + d[0], feature[1] + d[1])
        if q in index:
            out.append(4 * index[q] + Direction.DIRECTION_TO_INDEX[Direction.OPPOSITE_DIRECTIONS[d]])
    return out


def plan_table(cl):
    """uint16 [n, n] with n = 4 * floor cells: entry [s, g] = (cost << 3) | first action of ``MotionPlanner.get_plan(s,
    g)``, PLAN_UNREACHABLE where g is not reachable from s.  cost = path length + 1 for the final INTERACT; s == g is
    ``[INTERACT]`` at cost 1.  The path is ``Graph.get_node_path`` (search.py): from each node the first successor, in
    node order, that lies one step closer to the goal; its first action is the move or turn into that successor
    (``action_plan_from_positions``: only the last node of a shortest path can be a turn in place, and a turn toward
    the goal's orientation is the action of that edge)."""
    _, succ = motion_graph(cl)
    n = succ.shape[0]
    inf = np.iinfo(np.int32).max
    dist = np.full((n, n), inf, np.int32)
    for s in range(n):
        row = dist[s]
        row[s] = 0
        q = deque([s])
        while q:
            u = q.popleft()
            for v in succ[u]:
                if row[v] == inf:
                    row[v] = row[u] + 1
                    q.append(v)
    plan = np.full((n, n), PLAN_UNREACHABLE, np.uint16)
    for s in range(n):
        children = sorted(set(int(v) for v in succ[s]) - {s})
        action = {int(succ[s, a]): a for a in range(4)}
        closer = dist[children] < dist[s][None, :]  # [k, n]
        first = np.argmax(closer, axis=0)
        reach = dist[s] < inf
        acts = np.array([action[c] for c in children], np.int32)[first]
        ent = ((dist[s].astype(np.int64) + 1) << 3) | acts
        plan[s, reach] = ent[reach].astype(np.uint16)
    np.fill_diagonal(plan, (1 << 3) | A_INTERACT)
    return plan


def greedy_table(cl):
    """(one GREEDY_LAYOUT_DTYPE record, its plan table): the goal lists of ``MediumLevelActionManager`` (planners.py)
    in the order ``_get_ml_actions_for_positions`` builds them — features in ``terrain_pos_dict`` order, each feature's
    motion goals in N, S, E, W order — and go_to_closest_feature_actions' features (onion dispensers, tomato dispensers,
    pots, dish dispensers), whose first cheapest goal is the reference's (min_cost_to_feature keeps the first cheapest
    feature; the first cheapest goal of that feature is then the first cheapest goal of the list).  Counters hold no
    goal: NO_COUNTERS_PARAMS has no counter goals, so MotionPlanner.is_valid_motion_goal refuses every goal facing a
    counter and the objects on counters never enter a goal set."""
    check_layout(cl)
    plan = plan_table(cl)
    rec = np.zeros((), GREEDY_LAYOUT_DTYPE)
    rec["n_nodes"] = plan.shape[0]
    fi = np.full(256, 0xFF, np.uint8)
    for i, p in enumerate(cl.terrain_pos_dict[" "]):
        fi[L.pos_byte(p)] = i
    rec["free_index"] = fi
    rec["partial_order"] = cl.partial_pot_order()

    def goals(features):
        return [g for f in features for g in motion_goals(cl, f)]

    T = cl.terrain_pos_dict
    lists = [goals(T["O"]), goals(T["D"]), goals(T["S"]), goals(T["O"] + T["T"] + T["P"] + T["D"])]
    lists += [goals([cl.pot_locations[k]]) if k < cl.n_pots else [] for k in range(L.MAX_POTS)]
    flat = [g for lst in lists for g in lst]
    assert len(flat) <= MAX_GOALS
    rec["list_start"] = np.cumsum([0] + [len(lst) for lst in lists])
    rec["goal"][:len(flat)] = flat
    return rec, plan


def build_greedy_tables(layouts):
    """(tables uint8 [n_layouts, 2660], plans uint16 [sum of n_nodes^2]): each layout's record with ``plan_offset`` the
    index of its plan table's entry [0, 0] in ``plans``."""
    recs, plans, off = [], [], 0
    for cl in layouts:
        rec, plan = greedy_table(cl)
        rec["plan_offset"] = off
        off += plan.size
        recs.append(rec)
        plans.append(plan.reshape(-1))
    return np.stack(recs).view(np.uint8).reshape(len(layouts), -1), np.concatenate(plans)
