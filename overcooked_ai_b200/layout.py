"""Layout compiler: a layout description -> the device constant table + packed start record.

Inputs are the reference's layout FORMAT (a dict with a ``grid`` of rows plus recipe / order /
reward-shaping parameters — src/overcooked_ai_py/data/layouts/*.layout, read by
OvercookedGridworld.from_layout_name, overcooked_mdp.py:1151-1222).  Outputs follow
include/ovc_b200.h: one ``ovc_layout_t`` per layout, the packed int32 state record, and the
per-(cell, orientation) lookup that featurize_state needs.

Everything here runs once per layout on the host; none of it is on the per-step path.
"""
import ast
import json
import os
from collections import deque

import numpy as np

from overcooked_ai_b200.actions import Direction
from overcooked_ai_b200.state import (
    MAX_NUM_INGREDIENTS,
    ONION,
    TOMATO,
    ObjectState,
    OvercookedState,
    PlayerState,
    Recipe,
    SoupState,
)

# ---- constants shared with include/ovc_b200.h -------------------------------------------------
T_FLOOR, T_COUNTER, T_ONION, T_TOMATO, T_DISH, T_POT, T_SERVE, T_OUTSIDE = range(8)
TERRAIN_CODE = {" ": T_FLOOR, "X": T_COUNTER, "O": T_ONION, "T": T_TOMATO, "D": T_DISH, "P": T_POT, "S": T_SERVE}
O_NONE, O_ONION, O_TOMATO, O_DISH, O_SOUP = range(5)
OBJ_CODE = {"onion": O_ONION, "tomato": O_TOMATO, "dish": O_DISH, "soup": O_SOUP}
OBJ_NAME = {v: k for k, v in OBJ_CODE.items()}
OBJ_MASK = 0x3FFFFF
MAX_TICK = 16382
MAX_POTS = 4
MAX_SLOTS = 124
MAX_FREE = 128
NO_SLOT = 0xFF
LAYOUT_OLD_DYNAMICS = 1
SUPPORTED_STATE_WORDS = (16, 32, 64, 128)

BASE_REW_SHAPING_PARAMS = {  # overcooked_mdp.py:1018-1025
    "PLACEMENT_IN_POT_REW": 3,
    "DISH_PICKUP_REWARD": 3,
    "SOUP_PICKUP_REWARD": 5,
    "DISH_DISP_DISTANCE_REW": 0,
    "POT_DISTANCE_REW": 0,
    "SOUP_DISTANCE_REW": 0,
}

EVENT_TYPES = [  # overcooked_mdp.py:1027-1058 — bit i of the event mask is EVENT_TYPES[i]
    "tomato_pickup", "useful_tomato_pickup", "tomato_drop", "useful_tomato_drop", "potting_tomato",
    "onion_pickup", "useful_onion_pickup", "onion_drop", "useful_onion_drop", "potting_onion",
    "dish_pickup", "useful_dish_pickup", "dish_drop", "useful_dish_drop",
    "soup_pickup", "soup_delivery", "soup_drop",
    "optimal_onion_potting", "optimal_tomato_potting", "viable_onion_potting", "viable_tomato_potting",
    "catastrophic_onion_potting", "catastrophic_tomato_potting", "useless_onion_potting", "useless_tomato_potting",
]
EV_RECIPE_SHIFT = 25
EVF_STEPPED_DONE = 1 << 30

LAYOUT_DTYPE = np.dtype(
    [
        ("width", "<i4"), ("height", "<i4"), ("n_pots", "<i4"), ("n_slots", "<i4"), ("flags", "<i4"),
        ("rew_placement_in_pot", "<i4"), ("rew_dish_pickup", "<i4"), ("rew_soup_pickup", "<i4"),
        ("state_words", "<i4"), ("n_free", "<i4"), ("reserved", "<i4", (6,)),
        ("cook_time", "<i4", (16,)), ("deliver_value", "<i4", (16,)), ("best_value", "<i4", (16,)),
        ("cell", "<u2", (256,)), ("slot_pos", "u1", (128,)), ("free_pos", "u1", (128,)),
    ]
)
assert LAYOUT_DTYPE.itemsize == 1024

FEAT_LUT_DTYPE = np.dtype(
    [("d_onion", "i1", (2,)), ("d_tomato", "i1", (2,)), ("d_dish", "i1", (2,)), ("d_serve", "i1", (2,)),
     ("pot_order", "u1", (MAX_POTS,))]
)
assert FEAT_LUT_DTYPE.itemsize == 12

POTENTIAL_CONSTANTS = {  # overcooked_mdp.py:1060-1073
    "default": {"max_delivery_steps": 10, "max_pickup_steps": 10, "pot_onion_steps": 10, "pot_tomato_steps": 10},
    "mdp_test_tomato": {"max_delivery_steps": 4, "max_pickup_steps": 4, "pot_onion_steps": 5, "pot_tomato_steps": 6},
}

POTENTIAL_DTYPE = np.dtype(
    [
        ("steady", "<f8"), ("disc_value", "<f8", (16,)), ("opt_recipe", "<i4", (16,)),
        ("max_delivery_steps", "<i4"), ("max_pickup_steps", "<i4"), ("pot_onion_steps", "<i4"), ("pot_tomato_steps", "<i4"),
        ("onion_value", "<i4"), ("tomato_value", "<i4"), ("reserved", "<i4", (2,)),
        ("partial_order", "u1", (81, 4)), ("pad", "u1", (4,)),
    ]
)
assert POTENTIAL_DTYPE.itemsize == 560

COST_LUT_DTYPE = np.dtype([("serve", "u1"), ("pot", "u1", (MAX_POTS,)), ("pad", "u1", (3,))])
assert COST_LUT_DTYPE.itemsize == 8
COST_INF = 255

_DATA = os.path.join(os.path.dirname(__file__), "data", "layouts.json")
_LAYOUTS = None

RECIPE_CONFIG_KEYS = (
    "cook_time", "delivery_reward", "recipe_values", "recipe_times",
    "onion_value", "tomato_value", "onion_time", "tomato_time",
)


def pos_byte(pos):
    return (int(pos[1]) << 4) | int(pos[0])


def byte_pos(b):
    return (b & 15, b >> 4)


def layout_names():
    global _LAYOUTS
    if _LAYOUTS is None:
        with open(_DATA) as f:
            _LAYOUTS = json.load(f)
    return sorted(_LAYOUTS)


def read_layout_dict(layout_name):
    """Same role as the reference's utils.read_layout_dict (utils.py:223-226).  ``layout_name``
    is a bundled name, or a path to a reference-format ``.layout`` file (a dict literal)."""
    layout_names()
    if layout_name in _LAYOUTS:
        return json.loads(json.dumps(_LAYOUTS[layout_name]))
    path = layout_name if layout_name.endswith(".layout") else layout_name + ".layout"
    if os.path.exists(path):
        with open(path) as f:
            d = ast.literal_eval(f.read().replace("float('inf')", "1e999"))
        d["grid"] = [row.strip() for row in d["grid"].split("\n")]
        return d
    raise FileNotFoundError("unknown layout %r" % (layout_name,))


# ---- recipe tables ------------------------------------------------------------------------------
def _recipe_from_order(order):
    return order if isinstance(order, Recipe) else Recipe.from_dict(order)


def _resolve(conf, recipe, scalar_key, map_key, onion_key, tomato_key):
    """Recipe.value / Recipe.time resolution order, overcooked_mdp.py:136-188, including its
    truthiness tests (a 0 override falls through to the next rule)."""
    if conf.get(scalar_key):
        return conf[scalar_key]
    if conf.get(map_key):
        mapping = {}
        for order, v in zip(conf["all_orders"], conf[map_key]):
            mapping[_recipe_from_order(order)] = v
        if recipe in mapping:
            return mapping[recipe]
    if conf.get(onion_key) and conf.get(tomato_key):
        n_o, n_t = recipe.counts
        return conf[tomato_key] * n_t + conf[onion_key] * n_o
    return 20


def _check_recipe_config(conf):
    """The validity rules of Recipe.configure (overcooked_mdp.py:236-300): ValueError for a half-specified
    ingredient pair, for two mechanisms setting the same quantity, and for per-recipe lists that do not line
    up with the order list.  Like the reference, the rules look at which KEYS are present."""
    for kind in ("time", "value"):
        if ("tomato_" + kind in conf) != ("onion_" + kind in conf):
            raise ValueError("Must specify both 'onion_%s' and 'tomato_%s'" % (kind, kind))
    for ingredient_key, scalar_key, list_key in (("tomato_value", "delivery_reward", "recipe_values"),
                                                 ("tomato_time", "cook_time", "recipe_times")):
        for a, b in ((ingredient_key, scalar_key), (ingredient_key, list_key), (list_key, scalar_key)):
            if a in conf and b in conf:
                raise ValueError("%r is incompatible with %r" % (b, a))
        if list_key in conf:
            if not conf.get("all_orders"):
                raise ValueError("Must specify 'all_orders' if %r is specified" % list_key)
            if len(conf["all_orders"]) != len(conf[list_key]):
                raise ValueError("Number of recipes in 'all_orders' must be the same as number in %r" % list_key)


def _as_int(v, what):
    if isinstance(v, bool) or not (isinstance(v, (int, np.integer)) or (isinstance(v, float) and v.is_integer())):
        raise ValueError(
            "%s = %r is not an integer: the engine's reward / timer outputs are int32 "
            "(SURVEY.md appendix F)" % (what, v)
        )
    return int(v)


def assert_valid_grid(grid):
    """The grid rules of OvercookedGridworld._assert_valid_grid (overcooked_mdp.py:2064-2115), AssertionError like the
    reference and checked in its order: not ragged; no free cell (or player) on the border; players numbered
    1..n without gaps; known characters only; at least one dish dispenser, serving cell, pot and ingredient dispenser."""
    width = len(grid[0])
    assert all(len(row) == width for row in grid), "Ragged grid"
    solid = "XOPDST"
    for row in grid:
        assert row[0] in solid, "Left border must not be free"
        assert row[-1] in solid, "Right border must not be free"
    for x in range(width):
        assert grid[0][x] in solid, "Top border must not be free"
        assert grid[-1][x] in solid, "Bottom border must not be free"
    cells = [c for row in grid for c in row]
    digits = sorted(int(c) for c in cells if c in "123456789")
    assert len(digits) > 0, "No players (digits) in grid"
    assert digits == list(range(1, len(digits) + 1)), "Some players were missing"
    assert all(c in "XOPDST123456789 " for c in cells), "Invalid character in grid"
    assert cells.count("1") == 1, "'1' must be present exactly once"
    assert cells.count("D") >= 1, "'D' must be present at least once"
    assert cells.count("S") >= 1, "'S' must be present at least once"
    assert cells.count("P") >= 1, "'P' must be present at least once"
    assert cells.count("O") >= 1 or cells.count("T") >= 1, "'O' or 'T' must be present at least once"


class CompiledLayout(object):
    """One layout, compiled.  Attributes mirror what the reference's OvercookedGridworld keeps
    (terrain_mtx, start_player_positions, start_all_orders, ... overcooked_mdp.py:1090-1148)."""

    def __init__(self, layout_name, grid, start_all_orders=(), start_bonus_orders=(), rew_shaping_params=None,
                 order_bonus=2, old_dynamics=False, start_state=None, num_items_for_soup=3, **recipe_kwargs):
        self.layout_name = layout_name
        grid = [list(row) for row in grid]
        self.height, self.width = len(grid), len(grid[0])
        assert_valid_grid(grid)
        if self.width > 16 or self.height > 16:
            raise ValueError("grid %dx%d exceeds the 16x16 pos-byte range" % (self.width, self.height))
        players = {}
        for y, row in enumerate(grid):
            for x, c in enumerate(row):
                if c.isdigit() and c != "0":
                    players[int(c) - 1] = (x, y)
                    row[x] = " "
                elif c not in TERRAIN_CODE:
                    raise ValueError("Invalid character %r in grid" % c)
        self.start_player_positions = [players[i] for i in range(len(players))]
        self.num_players = len(players)
        if self.num_players != 2:
            raise ValueError(
                "layout %r has %d players; the batched engine implements the 2-player game "
                "(lossless_state_encoding itself asserts this, overcooked_mdp.py:2389-2391)"
                % (layout_name, self.num_players)
            )
        self.terrain_mtx = grid
        self.old_dynamics = bool(old_dynamics)
        self.order_bonus = order_bonus
        self.reward_shaping_params = dict(BASE_REW_SHAPING_PARAMS if rew_shaping_params is None else rew_shaping_params)
        self.start_bonus_orders = list(start_bonus_orders)
        self.recipe_config = dict(num_items_for_soup=num_items_for_soup, all_orders=list(start_all_orders))
        unknown = set(recipe_kwargs) - set(RECIPE_CONFIG_KEYS)
        if unknown:
            raise ValueError("unknown layout parameters %s" % sorted(unknown))
        self.recipe_config.update(recipe_kwargs)
        all_recipes = Recipe.all_recipes()
        # empty start_all_orders means "every recipe" (overcooked_mdp.py:1116-1120)
        self.start_all_orders = (
            [r.to_dict() for r in all_recipes] if not start_all_orders else list(start_all_orders)
        )
        if self.old_dynamics:
            assert all(len(o["ingredients"]) == 3 for o in self.start_all_orders), \
                "Only accept orders with 3 items when using the old_dynamics"

        # ---- terrain, slots ----
        self.terrain_pos_dict = {c: [] for c in TERRAIN_CODE}
        for y, row in enumerate(grid):
            for x, c in enumerate(row):
                self.terrain_pos_dict[c].append((x, y))
        self.pot_locations = list(self.terrain_pos_dict["P"])
        self.counter_locations = list(self.terrain_pos_dict["X"])
        self.slot_positions = self.pot_locations + self.counter_locations
        self.slot_of = {p: i for i, p in enumerate(self.slot_positions)}
        self.n_pots, self.n_slots = len(self.pot_locations), len(self.slot_positions)
        if self.n_pots > MAX_POTS:
            raise ValueError("layout %r has %d pots (max %d)" % (layout_name, self.n_pots, MAX_POTS))
        if self.n_slots > MAX_SLOTS:
            raise ValueError("layout %r has %d object cells (max %d)" % (layout_name, self.n_slots, MAX_SLOTS))
        if len(self.terrain_pos_dict[" "]) > MAX_FREE:  # free_pos[128] of the table: random start positions draw from it
            raise ValueError("layout %r has %d floor cells (max %d)" % (layout_name, len(self.terrain_pos_dict[" "]), MAX_FREE))
        self.state_words = next(s for s in SUPPORTED_STATE_WORDS if s >= 4 + self.n_slots)

        # ---- recipe tables ----
        conf = self.recipe_config
        _check_recipe_config(conf)
        all_set = set(_recipe_from_order(o) for o in self.start_all_orders)
        bonus_set = set(_recipe_from_order(o) for o in self.start_bonus_orders)
        self.cook_time = np.zeros(16, np.int64)
        self.base_value = np.zeros(16, np.int64)
        self.deliver_value = np.zeros(16, np.int64)
        for r in all_recipes:
            t = _as_int(_resolve(conf, r, "cook_time", "recipe_times", "onion_time", "tomato_time"), "cook time")
            v = _resolve(conf, r, "delivery_reward", "recipe_values", "onion_value", "tomato_value")
            if not 0 < t <= MAX_TICK:
                raise ValueError("cook time %d outside 1..%d" % (t, MAX_TICK))
            self.cook_time[r.index] = t
            self.base_value[r.index] = _as_int(v, "recipe value")
            if r in all_set:  # get_recipe_value, overcooked_mdp.py:1595-1602
                dv = v * order_bonus if r in bonus_set else v
                self.deliver_value[r.index] = _as_int(dv, "delivery reward of %r" % (r,))
        # best reachable delivery value from each partial recipe (DFS of :1976-2016 ends on the max)
        self.best_value = np.zeros(16, np.int64)
        for idx in range(16):
            o, t = idx >> 2, idx & 3
            if o + t > MAX_NUM_INGREDIENTS:
                continue
            reach = [
                self.deliver_value[oo * 4 + tt]
                for oo in range(o, 4) for tt in range(t, 4)
                if 0 < oo + tt <= MAX_NUM_INGREDIENTS
            ]
            best = max(reach)
            # the DFS keeps the start recipe when nothing beats 0 (:1988-2008)
            self.best_value[idx] = best if best > 0 else (self.deliver_value[idx] if idx else 0)

        # ---- start state ----
        if start_state is not None and not isinstance(start_state, OvercookedState):
            start_state = OvercookedState.from_dict(start_state)
        self.start_state = start_state

    # -- reference-compatible accessors -------------------------------------------------------
    def get_terrain_type_at_pos(self, pos):
        return self.terrain_mtx[pos[1]][pos[0]]

    def get_standard_start_state(self):
        """overcooked_mdp.py:1297-1305"""
        if self.start_state is not None:
            return self._with_cook_times(self.start_state.deepcopy())
        return OvercookedState.from_player_positions(
            self.start_player_positions, bonus_orders=self.start_bonus_orders, all_orders=self.start_all_orders
        )

    def soup_cook_time(self, soup):
        n_t = soup.ingredients.count(TOMATO)
        return int(self.cook_time[(len(soup.ingredients) - n_t) * 4 + n_t])

    def _with_cook_times(self, state):
        for obj in list(state.objects.values()) + [p.held_object for p in state.players if p.held_object]:
            if obj.name == "soup" and len(obj.ingredients) > 0:
                obj._cook_time = self.soup_cook_time(obj)
        return state

    # -- table for the device ------------------------------------------------------------------
    def table(self):
        rec = np.zeros((), LAYOUT_DTYPE)
        rec["width"], rec["height"] = self.width, self.height
        rec["n_pots"], rec["n_slots"] = self.n_pots, self.n_slots
        rec["flags"] = LAYOUT_OLD_DYNAMICS if self.old_dynamics else 0
        rsp = self.reward_shaping_params
        rec["rew_placement_in_pot"] = _as_int(rsp["PLACEMENT_IN_POT_REW"], "PLACEMENT_IN_POT_REW")
        rec["rew_dish_pickup"] = _as_int(rsp["DISH_PICKUP_REWARD"], "DISH_PICKUP_REWARD")
        rec["rew_soup_pickup"] = _as_int(rsp["SOUP_PICKUP_REWARD"], "SOUP_PICKUP_REWARD")
        rec["state_words"] = self.state_words
        rec["cook_time"] = self.cook_time
        rec["deliver_value"] = self.deliver_value
        rec["best_value"] = self.best_value
        cell = np.full(256, T_OUTSIDE | (NO_SLOT << 8), np.uint16)
        for y, row in enumerate(self.terrain_mtx):
            for x, c in enumerate(row):
                cell[pos_byte((x, y))] = TERRAIN_CODE[c] | (self.slot_of.get((x, y), NO_SLOT) << 8)
        rec["cell"] = cell
        sp = np.zeros(128, np.uint8)
        for i, p in enumerate(self.slot_positions):
            sp[i] = pos_byte(p)
        rec["slot_pos"] = sp
        free = self.terrain_pos_dict[" "]
        rec["n_free"] = len(free)
        fp = np.zeros(128, np.uint8)
        for i, p in enumerate(free):
            fp[i] = pos_byte(p)
        rec["free_pos"] = fp
        return rec

    # -- planner distances ------------------------------------------------------------------------
    def _bfs(self):
        """For every (free cell, orientation) start: BFS distances over (cell, orientation) nodes.

        Restates the motion-planner graph of the reference for the default NO_COUNTERS_PARAMS
        (planning/planners.py:27-34): edges are the four direction actions (move if the target is floor,
        else turn in place — _move_if_direction, overcooked_mdp.py:1718-1727; graph at planners.py:315-358);
        the goals of a feature cell f are (f+d, opposite(d)) for d in N,S,E,W order when f+d is floor
        (planners.py:439-450); counters are never goals.  Yields (start, orientation index, dist, goals_of).
        """
        free = [p for p in self.terrain_pos_dict[" "]]
        free_set = set(free)
        dirs = Direction.ALL_DIRECTIONS

        def goals_of(f):
            out = []
            for d in dirs:
                adj = (f[0] + d[0], f[1] + d[1])
                if adj in free_set:
                    out.append((adj, Direction.DIRECTION_TO_INDEX[Direction.OPPOSITE_DIRECTIONS[d]]))
            return out

        for start in free:
            for so in range(4):
                dist = {(start, so): 0}
                q = deque([(start, so)])
                while q:
                    (p, o) = q.popleft()
                    for a, d in enumerate(dirs):
                        np_ = (p[0] + d[0], p[1] + d[1])
                        nxt = (np_, a) if np_ in free_set else (p, a)
                        if nxt not in dist:
                            dist[nxt] = dist[(p, o)] + 1
                            q.append(nxt)
                yield start, so, dist, goals_of

    @staticmethod
    def _closest(dist, goals_of, features, exclude=()):
        """MotionPlanner.min_cost_to_feature (planners.py:391-423): (cost, feature); the first minimum in
        (feature order, direction order) wins; cost = distance + 1 for the interact; (None, None) if unreachable."""
        best, best_f = None, None
        for f in features:
            if f in exclude:
                continue
            for g in goals_of(f):
                if g in dist and (best is None or dist[g] < best):
                    best, best_f = dist[g], f
        return (None if best is None else best + 1), best_f

    def feature_lut(self):
        """featurize_state lookup: per (cell, orientation), deltas to the closest onion / tomato / dish
        dispenser and serving cell, and the pots ordered by planner cost."""
        lut = np.zeros((256, 4), FEAT_LUT_DTYPE)
        lut["pot_order"] = NO_SLOT
        for start, so, dist, goals_of in self._bfs():
            e = lut[pos_byte(start), so]
            for key, terr in (("d_onion", "O"), ("d_tomato", "T"), ("d_dish", "D"), ("d_serve", "S")):
                _, f = self._closest(dist, goals_of, self.terrain_pos_dict[terr])
                if f is not None:
                    e[key] = (f[0] - start[0], f[1] - start[1])
            taken = []
            for k in range(self.n_pots):
                _, f = self._closest(dist, goals_of, self.pot_locations, exclude=taken)
                if f is None:
                    break
                taken.append(f)
                e["pot_order"][k] = self.slot_of[f]
        return lut

    def cost_lut(self):
        """potential_function lookup: per (cell, orientation), min_cost_to_feature to the serving cells and
        to each pot (COST_INF = unreachable)."""
        lut = np.zeros((256, 4), COST_LUT_DTYPE)
        lut["serve"], lut["pot"] = COST_INF, COST_INF
        for start, so, dist, goals_of in self._bfs():
            e = lut[pos_byte(start), so]
            c, _ = self._closest(dist, goals_of, self.terrain_pos_dict["S"])
            if c is not None:
                e["serve"] = min(c, COST_INF - 1)
            for k, pot in enumerate(self.pot_locations):
                c, _ = self._closest(dist, goals_of, [pot])
                if c is not None:
                    e["pot"][k] = min(c, COST_INF - 1)
        return lut

    # -- potential_function constants -----------------------------------------------------------
    def potential_params(self):
        """overcooked_mdp.py:2972-2982 (onion / tomato value default to 21 / 13 when the layout has none)."""
        conf = self.recipe_config
        p = dict(POTENTIAL_CONSTANTS.get(self.layout_name, POTENTIAL_CONSTANTS["default"]))
        p["tomato_value"] = conf.get("tomato_value") if conf.get("tomato_value") else 13
        p["onion_value"] = conf.get("onion_value") if conf.get("onion_value") else 21
        return p

    def potential_table(self, gamma=0.99):
        """Per-layout constants of potential_function (overcooked_mdp.py:2920-3250) for a given gamma: the
        discounted best-recipe search (DFS of :1976-2016 with the discounted value of :1603-1629, whose
        visiting order decides ties), the steady-state term (:2985-2999) and CPython's iteration order of
        the set built by get_partially_full_pots (:1882-1890), which fixes the order idle soups are visited."""
        pp = self.potential_params()
        all_recipes = {r.index: r for r in Recipe.all_recipes()}

        def disc_value(idx, base_idx):
            o, t = idx >> 2, idx & 3
            bo, bt = (base_idx >> 2, base_idx & 3) if base_idx else (0, 0)
            n_on, n_to = o - bo, t - bt
            return (gamma ** int(self.cook_time[idx]) * gamma ** (pp["pot_onion_steps"] * n_on)
                    * gamma ** (pp["pot_tomato_steps"] * n_to) * int(self.deliver_value[idx]))

        def neighbors(idx):
            o, t = idx >> 2, idx & 3
            if o + t == MAX_NUM_INGREDIENTS:
                return []
            return [((o + 1) << 2) | t, (o << 2) | (t + 1)]  # ALL_INGREDIENTS order: onion, tomato (:201-204)

        rec = np.zeros((), POTENTIAL_DTYPE)
        for start in [0] + sorted(all_recipes):
            stack = [4, 1] if start == 0 else [start]  # [onion], [tomato] pushed in that order (:1991-1992)
            visited, best_idx, best_val = set(), start, 0
            while stack:
                cur = stack.pop()
                if cur in visited:
                    continue
                visited.add(cur)
                v = disc_value(cur, start)
                if v > best_val:
                    best_val, best_idx = v, cur
                for nb in neighbors(cur):
                    if nb not in visited:
                        stack.append(nb)
            rec["opt_recipe"][start] = best_idx
            rec["disc_value"][start] = best_val
        opt = int(rec["opt_recipe"][0])
        opt_value = int(self.deliver_value[opt]) if opt else 0
        if opt_value <= 0:
            raise ValueError("potential_function needs a recipe with a positive value (overcooked_mdp.py:2996-2998)")
        discount = float(rec["disc_value"][0]) / opt_value
        rec["steady"] = (discount / (1 - discount)) * opt_value
        for k in ("max_delivery_steps", "max_pickup_steps", "pot_onion_steps", "pot_tomato_steps", "onion_value", "tomato_value"):
            rec[k] = _as_int(pp[k], k)
        rec["partial_order"] = self.partial_pot_order()
        return rec

    def partial_pot_order(self):
        """uint8 [81, 4]: the order of list(set().union(one_item_pots, two_item_pots)) (get_partially_full_pots,
        overcooked_mdp.py:1882-1890) for every assignment of pots to classes: row sum_k class_k * 3^k (class 0 other, 1 one
        item, 2 two items), entries the pots' slots in CPython's set iteration order, NO_SLOT after the last."""
        order = np.full((81, 4), NO_SLOT, np.uint8)
        for code in range(3 ** self.n_pots):
            cls = [(code // 3 ** k) % 3 for k in range(self.n_pots)]
            ones = [self.pot_locations[k] for k in range(self.n_pots) if cls[k] == 1]
            twos = [self.pot_locations[k] for k in range(self.n_pots) if cls[k] == 2]
            for j, pos in enumerate(list(set().union(*[ones, twos]))):
                order[code, j] = self.slot_of[pos]
        return order

    def potential_pow_len(self):
        pp = self.potential_params()
        return int(self.cook_time.max() + pp["max_delivery_steps"] + pp["max_pickup_steps"]
                   + 3 * max(pp["pot_onion_steps"], pp["pot_tomato_steps"]) + 8)


def compile_layout(layout_name, **params_to_overwrite):
    """from_layout_name (overcooked_mdp.py:1151-1172): bundled or on-disk layout + overrides."""
    d = read_layout_dict(layout_name)
    grid = d.pop("grid")
    d.update(params_to_overwrite)
    d.pop("layout_name", None)
    return CompiledLayout(layout_name, grid, **d)


# ---- packed record <-> OvercookedState -----------------------------------------------------------
def pack_object(obj):
    """ObjectState / SoupState -> 22-bit object code (include/ovc_b200.h): the value types already ARE their codes."""
    if obj is None:
        return 0
    if not obj.code:
        raise KeyError(obj.name)
    if obj.code & 7 == O_SOUP and not obj.is_valid():
        raise ValueError("soup with %d ingredients" % len(obj.ingredients))
    return obj.code & OBJ_MASK


def unpack_object(code, position, layout=None):
    t = code & 7
    if t == O_NONE:
        return None
    if t != O_SOUP:
        return ObjectState(OBJ_NAME[t], position)
    soup = SoupState(position)
    soup.code = code & OBJ_MASK
    if layout is not None and (code >> 3) & 3:
        soup._cook_time = layout.soup_cook_time(soup)
    return soup


def pack_state(layout, state, layout_id=0, state_words=None, out=None):
    """OvercookedState -> int32[state_words] record.  Validates what _check_valid_state
    (overcooked_mdp.py:1910-1949) asserts, raising AssertionError like the reference."""
    S = layout.state_words if state_words is None else state_words
    assert S >= 4 + layout.n_slots, "state_words too small for this layout"
    rec = np.zeros(S, np.int64) if out is None else out
    rec[:] = 0
    assert len(state.players) == 2, "the engine implements the 2-player game"
    rec[0] = state.timestep
    seen = set()
    for i, p in enumerate(state.players):
        assert layout.get_terrain_type_at_pos(p.position) == " ", "player on terrain"
        assert p.position not in seen, "Overlapping players or objects"
        seen.add(p.position)
        held = p.held_object
        if held is not None:
            assert held.position == p.position
            assert held.is_valid()
        rec[1 + i] = pos_byte(p.position) | (Direction.DIRECTION_TO_INDEX[p.orientation] << 8) | (pack_object(held) << 10)
    dishes = 0
    for pos, obj in state.objects.items():
        assert obj.position == pos
        assert obj.is_valid()
        terr = layout.get_terrain_type_at_pos(pos)
        assert terr != " ", "loose object on the floor"
        if pos not in layout.slot_of:
            raise ValueError("object on a %r cell at %s: only counters and pots can hold objects" % (terr, pos))
        if terr == "P":
            assert obj.name == "soup", "object in pot is not a soup"
        elif obj.name == "dish":
            dishes += 1
        rec[4 + layout.slot_of[pos]] = pack_object(obj)
    rec[3] = (layout_id & 0xFF) | (dishes << 8)
    # orders are layout constants in this engine: refuse states that disagree with the layout
    if [r for r in state.all_orders] != sorted(Recipe.from_dict(o) for o in layout.start_all_orders) or \
            state.bonus_orders != sorted(Recipe.from_dict(o) for o in layout.start_bonus_orders):
        raise ValueError("state order lists differ from the layout's (orders are per-layout constants here)")
    if out is None:
        # bit 31 of a player word is the top bit of a held soup's tick: go through uint32
        return (rec & 0xFFFFFFFF).astype(np.uint32).view(np.int32)
    return rec


def unpack_state(layout, rec):
    """int32[state_words] record -> OvercookedState (soups get the layout's cook time)."""
    rec = [int(v) & 0xFFFFFFFF for v in rec]
    players = []
    for i in range(2):
        w = rec[1 + i]
        pos = byte_pos(w & 0xFF)
        held = unpack_object((w >> 10) & OBJ_MASK, pos, layout)
        players.append(PlayerState(pos, Direction.INDEX_TO_DIRECTION[(w >> 8) & 3], held))
    objects = {}
    for k, pos in enumerate(layout.slot_positions):
        obj = unpack_object(rec[4 + k] & OBJ_MASK, pos, layout)
        if obj is not None:
            objects[pos] = obj
    ts = rec[0] if rec[0] < (1 << 31) else rec[0] - (1 << 32)
    return OvercookedState(
        players, objects, bonus_orders=layout.start_bonus_orders, all_orders=layout.start_all_orders, timestep=ts
    )


def build_tables(layouts, state_words=None):
    """Stack compiled layouts: (table bytes as uint8 [n, 1024], start records int32 [n, S], S)."""
    S = max(l.state_words for l in layouts) if state_words is None else state_words
    assert S in SUPPORTED_STATE_WORDS and all(l.state_words <= S for l in layouts)
    assert len(layouts) <= 256
    tab = np.stack([l.table() for l in layouts])
    starts = np.stack([pack_state(l, l.get_standard_start_state(), i, S) for i, l in enumerate(layouts)])
    return tab.view(np.uint8).reshape(len(layouts), -1), starts.astype(np.int32), S


def build_potential_tables(layouts, gamma=0.99):
    """(pot tables uint8 [n, 560], cost LUT uint8 [n, 256*4*8], gamma powers float64 [n_pow])."""
    pt = np.stack([l.potential_table(gamma) for l in layouts]).view(np.uint8).reshape(len(layouts), -1)
    cl = np.stack([l.cost_lut() for l in layouts]).view(np.uint8).reshape(len(layouts), -1)
    n_pow = max(l.potential_pow_len() for l in layouts)
    gpow = np.array([gamma ** k for k in range(n_pow)], np.float64)  # Python float pow, as the reference computes it
    return pt, cl, gpow
