"""The host tables of the limit layouts (``limit_layouts.py``) against independent restatements, and the hand-built states
through pack / unpack and the oracle.  No GPU needed.

The oracle reads the host's own tables (``feature_lut``, ``cost_lut``, ``potential_table``), so a wrong table would be
wrong on both sides of every kernel-vs-oracle comparison.  For 3 and 4 pots these tests restate the tables from scratch."""
from collections import deque

import numpy as np
import pytest

import limit_layouts as LL
from helpers import lut_bytes
from oracle import cpu
from overcooked_ai_b200 import layout as L

DIRS = [(0, -1), (0, 1), (1, 0), (-1, 0)]  # N, S, E, W: action / orientation index order
OPP = {0: 1, 1: 0, 2: 3, 3: 2}


def limit_layouts():
    return [LL.l16(), LL.l16_old(), LL.l3p(), LL.thin_16x3(), LL.thin_3x16()] + [LL.k7_layouts(w, h, 1)[0] for w, h in ((13, 7), (7, 13), (12, 8))]


LAYOUTS = limit_layouts()
IDS = [l.layout_name for l in LAYOUTS]


def planner_costs(grid, start, ori):
    """BFS over (cell, orientation) from one start: a direction action moves onto floor, else turns in place.  Returns
    {(cell, orientation): number of actions}."""
    H, W = len(grid), len(grid[0])
    floor = lambda x, y: 0 <= x < W and 0 <= y < H and grid[y][x] in " 12"
    dist = np.full((W, H, 4), -1, np.int64)
    dist[start[0], start[1], ori] = 0
    q = deque([(start[0], start[1], ori)])
    while q:
        x, y, o = q.popleft()
        for a, (dx, dy) in enumerate(DIRS):
            nx, ny = (x + dx, y + dy) if floor(x + dx, y + dy) else (x, y)
            if dist[nx, ny, a] < 0:
                dist[nx, ny, a] = dist[x, y, o] + 1
                q.append((nx, ny, a))
    return dist


def feature_cost(grid, dist, f):
    """min_cost_to_feature for one feature cell (PLN:391-423): the cheapest of its goals (floor neighbour facing it, in
    N, S, E, W order) + 1 for the interact; None if no goal is reachable."""
    H, W = len(grid), len(grid[0])
    best = None
    for d, (dx, dy) in enumerate(DIRS):
        x, y = f[0] + dx, f[1] + dy
        if 0 <= x < W and 0 <= y < H and grid[y][x] in " 12" and dist[x, y, OPP[d]] >= 0:
            c = int(dist[x, y, OPP[d]]) + 1
            if best is None or c < best:
                best = c
    return best


def closest(grid, dist, feats):
    """(cost, feature): the first feature (in list order) of minimal cost, as the strict '<' of PLN:391-423 keeps it."""
    costs = [(feature_cost(grid, dist, f), i) for i, f in enumerate(feats)]
    costs = [(c, i) for c, i in costs if c is not None]
    if not costs:
        return None, None
    c, i = min(costs)
    return c, feats[i]


def restated_tables(lay):
    """(feature_lut, cost_lut) restated from the grid text alone."""
    grid = ["".join(r) for r in lay.terrain_mtx]
    cells = {c: [(x, y) for y, row in enumerate(grid) for x, ch in enumerate(row) if ch == c] for c in "OTDSP"}
    pots = cells["P"]
    flut = np.zeros((256, 4), L.FEAT_LUT_DTYPE)
    flut["pot_order"] = L.NO_SLOT
    clut = np.zeros((256, 4), L.COST_LUT_DTYPE)
    clut["serve"], clut["pot"] = L.COST_INF, L.COST_INF
    for y, row in enumerate(grid):
        for x, ch in enumerate(row):
            if ch != " ":
                continue
            for o in range(4):
                dist = planner_costs(grid, (x, y), o)
                e, c = flut[(y << 4) | x, o], clut[(y << 4) | x, o]
                for key, t in (("d_onion", "O"), ("d_tomato", "T"), ("d_dish", "D"), ("d_serve", "S")):
                    _, f = closest(grid, dist, cells[t])
                    if f is not None:
                        e[key] = (f[0] - x, f[1] - y)
                pc = [feature_cost(grid, dist, p) for p in pots]
                # pots by cost, ties in pot order (a stable sort == repeated first-minimum with the chosen pots excluded)
                order = sorted((k for k in range(len(pots)) if pc[k] is not None), key=lambda k: pc[k])
                for j, k in enumerate(order):
                    e["pot_order"][j] = k  # pots are the first slots, in pot_locations order
                    c["pot"][k] = min(pc[k], L.COST_INF - 1)
                sc, _ = closest(grid, dist, cells["S"])
                if sc is not None:
                    c["serve"] = min(sc, L.COST_INF - 1)
    return flut, clut


@pytest.mark.parametrize("what", sorted(LL.refused()))
def test_layouts_beyond_the_limits_are_refused_when_compiled(what):
    make, reason = LL.refused()[what]
    with pytest.raises(ValueError, match=reason):
        make()


def test_limit_layouts_reach_the_limits():
    l16, l3p = LL.l16(), LL.l3p()
    assert (l16.width, l16.height, l16.n_pots, l16.n_slots, l16.state_words) == (16, 16, 4, L.MAX_SLOTS, 128)
    assert len(l16.terrain_pos_dict[" "]) <= L.MAX_FREE
    assert {1, 255, 256, 257, L.MAX_TICK} <= set(l16.cook_time.tolist())
    assert l3p.n_pots == 3 and int(l3p.table()["n_free"]) == L.MAX_FREE
    for lay in (LL.thin_16x3(), LL.thin_3x16()):
        grid = lay.terrain_mtx
        assert max(lay.width, lay.height) == 16 and min(lay.width, lay.height) == 3
        # a floor cell next to the x = 15 / y = 15 edge
        assert any(grid[y][x] == " " and (x == 14 or y == 14) for y in range(lay.height) for x in range(lay.width))


@pytest.mark.parametrize("lay", LAYOUTS, ids=IDS)
def test_planner_tables_vs_independent_restatement(lay):
    flut, clut = restated_tables(lay)
    got_f, got_c = lay.feature_lut(), lay.cost_lut()
    for k in ("d_onion", "d_tomato", "d_dish", "d_serve", "pot_order"):
        assert np.array_equal(got_f[k], flut[k]), k
    for k in ("serve", "pot"):
        assert np.array_equal(got_c[k], clut[k]), k
    if lay.layout_name == "L16":  # the pots are spread out: their planner order changes across the grid
        orders = {tuple(r) for r in flut["pot_order"].reshape(-1, 4).tolist() if r[0] != L.NO_SLOT}
        assert len(orders) >= 8 and all(L.NO_SLOT not in r for r in orders)


@pytest.mark.parametrize("make", [LL.l16, LL.l3p], ids=["L16", "L3P"])
def test_partial_order_is_cpython_set_order_for_3_and_4_pots(make):
    lay = make()
    n = lay.n_pots
    order = lay.potential_table(0.99)["partial_order"]
    differs = 0
    for code in range(3 ** n):
        cls = [(code // 3 ** k) % 3 for k in range(n)]
        ones = [p for p, c in zip(lay.pot_locations, cls) if c == 1]
        twos = [p for p, c in zip(lay.pot_locations, cls) if c == 2]
        want = [lay.pot_locations.index(p) for p in list(set().union(ones, twos))]
        assert order[code, :len(want)].tolist() == want and (order[code, len(want):] == L.NO_SLOT).all(), code
        differs += want != sorted(want)
    assert (order[3 ** n:] == L.NO_SLOT).all()
    assert differs > 0, "set order equals pot order everywhere: the test would not see a pot-index order"


def test_gamma_power_table_covers_the_longest_cook_time():
    lay = LL.l16()
    pp = lay.potential_params()
    for gamma in (0.99, 0.9):
        _, _, gpow = L.build_potential_tables([lay], gamma)
        need = L.MAX_TICK + pp["max_delivery_steps"] + pp["max_pickup_steps"] + 3 * max(pp["pot_onion_steps"], pp["pot_tomato_steps"])
        assert len(gpow) > need
        k = np.array([0, 1, 255, 16382, len(gpow) - 1])
        assert np.array_equal(gpow[k], np.array([gamma ** int(i) for i in k]))


def _all_states():
    out = []
    for lay, states in ((LL.l16(), LL.l16_states), (LL.l16_old(), LL.l16_old_states), (LL.l3p(), LL.l3p_states)):
        for name, s in states(lay).items():
            out.append((lay, name, s))
    return out


def test_hand_built_states_round_trip_and_the_oracle_accepts_them():
    for lay, name, s in _all_states():
        rec = L.pack_state(lay, s)
        assert rec.shape == (128,) and rec.dtype == np.int32
        back = L.unpack_state(lay, rec)
        assert back == s, name
        assert np.array_equal(L.pack_state(lay, back), rec), name
        dishes = sum(1 for p, o in s.objects.items() if o.name == "dish")
        assert int(rec[3]) >> 8 == dishes
        if name == "held_16382":
            assert int(rec[1]) < 0  # bit 31 of the player word: the top bit of the held soup's tick
        if name == "all_slots":
            assert (rec[4:] != 0).all() and dishes > 0
        tab, starts, _ = L.build_tables([lay])
        st = np.repeat(rec[None], 3, 0)
        acts = np.array([[[5, 5]] * 3, [[4, 4]] * 3], np.int32)
        cpu.rollout(tab, starts, st.copy(), acts, horizon=0)
        enc = cpu.encode_lossless(tab, st, lay.width, lay.height, 400)
        assert enc.shape == (3, 2, 16, 16, 26)
        f = cpu.featurize(tab, lut_bytes([lay]), st, lay.n_pots)
        assert np.isfinite(f).all()
        pt, cl, gpow = L.build_potential_tables([lay], 0.99)
        assert np.isfinite(cpu.potential(tab, pt, cl, gpow, st)).all()


def test_oracle_pot_features_follow_the_restated_pot_order():
    """cpu.featurize's pot blocks (num_pots = 4) name the pots in the restated planner order, and over-cooked soups show the
    reference's cook time remaining clipped at 0."""
    lay = LL.l16()
    flut, _ = restated_tables(lay)
    tab, _, _ = L.build_tables([lay])
    recs = np.stack([L.pack_state(lay, s) for s in LL.l16_states(lay).values()])
    f = cpu.featurize(tab, lut_bytes([lay]), recs, 4)
    B = 10 * 4 + 26
    for i, rec in enumerate(recs):
        for j in range(2):
            w = int(rec[1 + j]) & 0xFFFFFFFF
            x, y, o = w & 15, (w >> 4) & 15, (w >> 8) & 3
            for k in range(4):
                slot = int(flut["pot_order"][(y << 4) | x, o][k])
                blk = f[i, j, 22 + 10 * k: 32 + 10 * k]
                assert slot != L.NO_SLOT and blk[0] == 1
                px, py = lay.slot_positions[slot]
                assert (blk[8], blk[9]) == (px - x, py - y)
                assert blk[7] >= 0
        assert f.shape[2] == 2 * B + 4
