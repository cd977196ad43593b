"""Layouts and hand-built states at the limits of what ``layout.CompiledLayout`` accepts: 16x16 grids, 4 pots, 124 object
cells (a 128-word record), 128 floor cells, cook times up to 16382 (``MAX_TICK``), and the grids around K7's
shared-memory limit.  Everything is deterministic; nothing is random at import."""
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.actions import Direction
from overcooked_ai_b200.state import ObjectState, OvercookedState, PlayerState, SoupState

N, S, E, W = Direction.NORTH, Direction.SOUTH, Direction.EAST, Direction.WEST
O3, OT, O1, O2, T1, T3 = (["onion"] * 3, ["onion", "tomato"], ["onion"], ["onion"] * 2, ["tomato"], ["tomato"] * 3)


def _orders(*recipes):
    return [{"ingredients": r} for r in recipes]


def _grid(width, height, border, interior):
    """A width x height grid of counters; ``border`` / ``interior``: {(x, y): char} placed on it (interior default floor)."""
    g = [["X"] * width for _ in range(height)]
    for y in range(1, height - 1):
        for x in range(1, width - 1):
            g[y][x] = " "
    for (x, y), c in list(border.items()) + list(interior.items()):
        g[y][x] = c
    return ["".join(r) for r in g]


# ---- L16: 16x16, 4 pots, 124 object cells (record of 128 words), 125 floor cells -----------------------------------------
def l16_grid(extra=None):
    border = {(0, 2): "P", (15, 13): "P", (6, 0): "P",
              (0, 13): "O", (13, 15): "O", (15, 4): "T", (3, 0): "D", (15, 8): "D", (12, 0): "S", (2, 15): "S"}
    interior = {(7, 13): "P", (1, 1): "1", (14, 14): "2"}
    for y in (2, 4, 6, 8, 10, 12):  # counter bars, open at both ends
        for x in range(3, 13):
            interior[(x, y)] = "X"
    for y in (3, 5, 7, 9, 11):  # single counters in the side corridors
        interior[(1, y)] = interior[(14, y)] = "X"
    border.update(extra or {})
    return _grid(16, 16, border, interior)


L16_TIMES = {"one onion": 1, "two onions": 255, "three onions": 256, "one tomato": 257, "onion + tomato": 16382, "three tomatoes": 100}
L16_PARAMS = dict(
    start_all_orders=_orders(O1, O2, O3, T1, OT, T3),
    recipe_times=[1, 255, 256, 257, 16382, 100],
    recipe_values=[3, 7, 20, 9, 40, 15],
    start_bonus_orders=_orders(O3),
    order_bonus=3,
    rew_shaping_params={"PLACEMENT_IN_POT_REW": 2, "DISH_PICKUP_REWARD": 7, "SOUP_PICKUP_REWARD": 11,
                        "DISH_DISP_DISTANCE_REW": 0, "POT_DISTANCE_REW": 0, "SOUP_DISTANCE_REW": 0},
)
# old dynamics takes 3-ingredient orders only
L16_OLD_PARAMS = dict(
    start_all_orders=_orders(O3, ["onion", "onion", "tomato"], ["onion", "tomato", "tomato"], T3),
    recipe_times=[256, 1, 257, 16382],
    recipe_values=[20, 5, 9, 40],
    start_bonus_orders=_orders(T3),
    old_dynamics=True,
)


def l16(name="L16", **over):
    return L.CompiledLayout(name, l16_grid(), **dict(L16_PARAMS, **over))


def l16_old():
    return L.CompiledLayout("L16_old", l16_grid(), **L16_OLD_PARAMS)


# ---- L3P: open 16x16 with exactly 128 floor cells and 3 pots (n_free at its limit) ------------------------------------------
def l3p_grid(extra_floor=0):
    border = {(3, 0): "P", (12, 0): "P", (0, 5): "P", (15, 3): "O", (0, 8): "T", (8, 0): "D", (15, 7): "S"}
    interior = {(1, 1): "1", (14, 9): "2"}
    for y in range(10, 15):
        for x in range(1, 15):
            interior[(x, y)] = "X"
    interior[(1, 10)] = interior[(14, 10)] = " "  # rows 1-9 are open: 126 + 2 = 128 floor cells
    for k in range(extra_floor):
        interior[(2 + k, 10)] = " "
    return _grid(16, 16, border, interior)


def l3p():
    return L.CompiledLayout("L3P", l3p_grid(), start_all_orders=_orders(O3, OT, T1), recipe_times=[300, 5, 16382],
                            start_bonus_orders=_orders(OT))


# ---- thin grids: 16x3 and 3x16 ----------------------------------------------------------------------------------------------
def thin_16x3():
    return L.CompiledLayout("thin_16x3", ["XXOXXXXXXXXXDXXX", "P1            2S", "XXXXXXPXXXXXXTXX"], cook_time=3)


def thin_3x16():
    rows = ["XPX", "X1X"] + ["X X"] * 12 + ["X2X", "XSX"]
    rows[3], rows[7], rows[10], rows[12] = "O X", "X P", "X D", "T X"
    return L.CompiledLayout("thin_3x16", rows, cook_time=3)


# ---- K7 shape edge: 13x7 / 7x13 (largest that fit), 12x8 (96 cells, smallest refused) ---------------------------------------
def k7_grid(width, height, variant=0):
    border = {(0, 1): "P", (width - 1, height - 2): "P", (width // 2, 0): "O", (1, height - 1): "D", (width - 2, 0): "S",
              (0, height - 2): "T"}
    interior = {(1, 1): "1", (width - 2, height - 2): "2"}
    for k in range(variant):  # a few counters change the planner's tables between variants
        interior[(2 + k, height // 2)] = "X"
    return _grid(width, height, border, interior)


def k7_layouts(width, height, n=8):
    """n layouts of one grid shape: one with a 16382-step soup, the others with other cook times / values / counters."""
    out = []
    for i in range(n):
        times = [16382, 3, 257] if i == 0 else [5 + i, 3 + 2 * i, 255 + i]
        out.append(L.CompiledLayout("k7_%dx%d_%d" % (width, height, i), k7_grid(width, height, i % 3),
                                    start_all_orders=_orders(O3, OT, T1), recipe_times=times, recipe_values=[20, 9 + i, 5]))
    return out


# ---- layouts beyond the limits: each must be refused when compiled ------------------------------------------------------------
def refused():
    """{what: (callable compiling it, pattern of the ValueError it must raise)}."""
    wide = [row[:9] + row[8] + row[9:] for row in l16_grid()]  # a 17th column (a copy of column 8)
    return {
        "17 wide": (lambda: L.CompiledLayout("wide", wide), "exceeds the 16x16 pos-byte range"),
        "5 pots": (lambda: L.CompiledLayout("pots5", l16_grid({(0, 6): "P"})), "has 5 pots"),
        "125 object cells": (lambda: L.CompiledLayout("slots125", l16_grid({(13, 15): "X"})), "has 125 object cells"),
        "129 floor cells": (lambda: L.CompiledLayout("free129", l3p_grid(extra_floor=1)), "has 129 floor cells"),
        "cook time 16383": (lambda: l16("cook16383", recipe_times=[1, 255, 256, 257, 16383, 100]), "cook time 16383 outside"),
    }


# ---- hand-built states ----------------------------------------------------------------------------------------------------------
def soup(pos, ingredients, tick):
    return SoupState(pos, [ObjectState(i, pos) for i in ingredients], tick)


def _state(lay, players, objects, timestep=0):
    ps = []
    for pos, ori, held in players:
        if isinstance(held, tuple):  # (ingredients, tick): a held soup
            held = soup(pos, *held)
        elif held is not None:
            held = ObjectState(held, pos)
        ps.append(PlayerState(pos, ori, held))
    objs = {o.position: o for o in objects}
    return OvercookedState(ps, objs, bonus_orders=lay.start_bonus_orders, all_orders=lay.start_all_orders, timestep=timestep)


def l16_states(lay):
    """{name: OvercookedState} on L16 (pots at (6,0), (0,2), (7,13), (15,13); cook times L16_TIMES)."""
    P0, P1, P2, P3 = (6, 0), (0, 2), (7, 13), (15, 13)
    st = {}
    # around the ready tick: cook - 1, cook, cook + 1 (over-cooked: hand-built only, K5's POT_FROZEN), 16382 - 1
    st["ticks"] = _state(lay, [((1, 2), W, "dish"), ((6, 1), N, "dish")],
                         [soup(P0, O3, 255), soup(P1, O3, 256), soup(P2, O3, 257), soup(P3, OT, 16381)])
    st["overcooked"] = _state(lay, [((6, 13), E, None), ((8, 13), W, "dish")],
                              [soup(P0, O2, 300), soup(P1, O1, 2), soup(P2, T1, 16382), soup(P3, OT, 16382)])
    # a held soup with tick 16382 sets bit 31 of the player word; player 0 faces the serving cell (2, 15)
    st["held_16382"] = _state(lay, [((2, 14), S, (OT, 16382)), ((6, 1), N, "onion")],
                              [soup(P0, OT, 0), soup(P1, O1, 1), soup(P2, O3, -1), soup(P3, T3, -1)])
    # all pots full (n_full = n_pots = 4), players at the onion and dish dispensers
    st["all_full"] = _state(lay, [((1, 13), W, None), ((3, 1), N, None)],
                            [soup(P0, O3, -1), soup(P1, OT, 0), soup(P2, O3, 10), soup(P3, T3, -1)])
    st["idle_full"] = _state(lay, [((1, 2), W, None), ((14, 13), E, None)],
                             [soup(P0, O3, -1), soup(P1, O3, -1), soup(P2, T3, -1), soup(P3, ["onion", "onion", "tomato"], -1)])
    # both players interact with pot (7, 13) in the same transition
    st["same_pot_add"] = _state(lay, [((6, 13), E, "onion"), ((8, 13), W, "onion")], [soup(P2, O2, -1)])
    st["same_pot_plate"] = _state(lay, [((6, 13), E, "dish"), ((8, 13), W, "dish")], [soup(P2, O1, 1), soup(P0, O3, 256)])
    # every one of the 124 slots occupied; word 3 counts the loose dishes
    objs = [soup(P0, O3, 100), soup(P1, O1, -1), soup(P2, OT, 5), soup(P3, O3, 256)]
    kinds = ["onion", "tomato", "dish", "soup"]
    for k, pos in enumerate(lay.counter_locations):
        name = kinds[k % 4]
        objs.append(soup(pos, [OT, O3, T1][k % 3], 16382) if name == "soup" else ObjectState(name, pos))  # plated soups are done
    st["all_slots"] = _state(lay, [((1, 1), N, None), ((14, 14), S, "dish")], objs, timestep=17)
    return st


def l16_old_states(lay):
    P0, P1, P2, P3 = (6, 0), (0, 2), (7, 13), (15, 13)
    return {"idle_full_old": _state(lay, [((1, 2), W, None), ((6, 13), E, "onion")],
                                    [soup(P0, O3, -1), soup(P1, ["onion", "onion", "tomato"], -1), soup(P2, O2, -1), soup(P3, T3, -1)])}


def l3p_states(lay):
    return {"ticks": _state(lay, [((3, 1), N, "dish"), ((1, 5), W, "onion")],
                            [soup((3, 0), O3, 299), soup((12, 0), OT, 5), soup((0, 5), T1, 16381)])}

