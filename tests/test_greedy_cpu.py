"""The greedy partner without a GPU: the host restatement (tests/greedy_reference.py) against the reference's own
GreedyHumanModel games (tests/golden/greedy_cramped_room.npz), the plan tables against a BFS of the motion graph, and the
library's kernels, exports and argument checks."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch
from types import SimpleNamespace

import greedy_reference as R
import test_gpu_greedy as GG
from helpers import GOLD, strip_signature
from overcooked_ai_b200 import _greedy_native, greedy as G
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN, SelfPlayRollout
from test_policy_forms_cpu import _tool, defined_tests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    d = np.load(GOLD + "/greedy_cramped_room.npz")
    return L.compile_layout("cramped_room"), d["states"], d["actions"]


def _stuck(states, e, t):
    return t > 0 and R.players_key(states[e, t - 1]) == R.players_key(states[e, t])


def test_restatement_reproduces_every_deterministic_golden_action():
    """5 x 400 steps of GreedyHumanModel self-play: at the 1 512 steps where the players moved or turned, both agents'
    actions (3 024) are the restatement's."""
    cl, states, actions = _golden()
    lp = R.LayoutPlanner(cl)
    checked = 0
    for e in range(states.shape[0]):
        for t in range(states.shape[1]):
            if _stuck(states, e, t):
                continue
            for p in range(2):
                assert R.planned_action(lp, states[e, t], p) == actions[e, t, p], (e, t, p)
                checked += 1
    assert checked == 3024


def test_every_stuck_golden_action_is_an_unblocking_move():
    """At the 488 stuck steps (both players' positions and orientations unchanged) the reference drew from numpy: each
    agent's action lies in the restatement's unblocking set."""
    cl, states, actions = _golden()
    lp = R.LayoutPlanner(cl)
    n = 0
    for e in range(states.shape[0]):
        for t in range(states.shape[1]):
            if _stuck(states, e, t):
                n += 1
                for p in range(2):
                    assert actions[e, t, p] in R.unblocking_actions(lp, states[e, t], p), (e, t, p)
    assert n == 488


def test_the_golden_has_no_object_but_soup_on_a_counter():
    """Why the counter-object goal order (record slot order here, insertion order in the reference) is never exercised
    by the golden."""
    cl, states, _ = _golden()
    counters = states[..., 4 + cl.n_pots:4 + cl.n_slots] & 7
    assert np.isin(counters, [L.O_NONE, L.O_SOUP]).all()


def qualifying_layouts():
    out = []
    for name in L.layout_names():
        try:
            cl = L.compile_layout(name)
            G.check_layout(cl)
        except (ValueError, AssertionError):
            continue
        out.append(cl)
    return out


def test_plan_costs_are_bfs_distance_plus_one_on_every_qualifying_layout():
    """Every plan entry against CompiledLayout._bfs (the featurisation's own BFS of the same graph): cost = distance + 1,
    unreachable exactly where the BFS does not reach, [INTERACT] at cost 1 on the diagonal; the first action leads to a
    node one step closer, and no successor earlier in node order does (Graph._get_next_node)."""
    layouts = qualifying_layouts()
    assert len(layouts) >= 20
    for cl in layouts:
        free, succ = G.motion_graph(cl)
        index = {p: i for i, p in enumerate(free)}
        plan = G.plan_table(cl)
        n = plan.shape[0]
        dist = np.full((n, n), -1, np.int64)
        for start, so, d, _ in cl._bfs():
            s = 4 * index[start] + so
            for (p, o), v in d.items():
                dist[s, 4 * index[p] + o] = v
        reach = dist >= 0
        assert np.array_equal(plan != G.PLAN_UNREACHABLE, reach), cl.layout_name
        cost, act = plan.astype(np.int64) >> 3, plan & 7
        assert np.array_equal(cost[reach], dist[reach] + 1), cl.layout_name
        assert (np.diag(act) == G.A_INTERACT).all()
        off = reach & ~np.eye(n, dtype=bool)
        s_idx, g_idx = np.nonzero(off)
        a = act[s_idx, g_idx]
        assert (a < 4).all()
        nxt = succ[s_idx, a]
        assert (dist[nxt, g_idx] == dist[s_idx, g_idx] - 1).all(), cl.layout_name
        for k in range(4):  # no closer successor earlier in node order
            other = succ[s_idx, k]
            earlier = (other < nxt) & (other != s_idx)
            assert not (earlier & (dist[other, g_idx] == dist[s_idx, g_idx] - 1)).any(), cl.layout_name


def test_layouts_without_one_three_onion_order_are_refused():
    for name in ("cramped_room_tomato", "bonus_order_test"):
        with pytest.raises(ValueError, match="one order of three onions"):
            G.greedy_table(L.compile_layout(name))
    with pytest.raises(ValueError, match="one order of three onions"):
        R.LayoutPlanner(L.compile_layout("cramped_room", start_all_orders=[{"ingredients": ["onion"] * 3},
                                                                           {"ingredients": ["onion"] * 2}]))


def test_greedy_table_matches_the_c_struct_and_its_lists():
    cl = next(c for c in qualifying_layouts() if c.n_pots >= 2)
    tab, plans = G.build_greedy_tables([L.compile_layout("cramped_room"), cl])
    assert tab.shape[1] == G.GREEDY_LAYOUT_DTYPE.itemsize == _greedy_native.lib().ovc_greedy_layout_table_size()
    recs = tab.view(G.GREEDY_LAYOUT_DTYPE).reshape(-1)
    assert recs[1]["plan_offset"] == recs[0]["n_nodes"] ** 2 and plans.size == sum(int(r["n_nodes"]) ** 2 for r in recs)
    r, T = recs[1], cl.terrain_pos_dict
    lst = lambda k: list(r["goal"][r["list_start"][k]:r["list_start"][k + 1]])
    goals = lambda cells: [g for c in cells for g in G.motion_goals(cl, c)]
    assert lst(G.LIST_ONION) == goals(T["O"]) and lst(G.LIST_DISH) == goals(T["D"]) and lst(G.LIST_SERVE) == goals(T["S"])
    assert lst(G.LIST_CLOSEST) == goals(T["O"] + T["T"] + T["P"] + T["D"])
    for k in range(L.MAX_POTS):
        assert lst(G.LIST_POT + k) == (goals([cl.pot_locations[k]]) if k < cl.n_pots else [])


def test_library_kernels_are_the_gpu_tests_table():
    """Every device entry point of libovc_greedy.so has a case in tests/test_gpu_greedy.py, and every listed one exists."""
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if not cuobjdump or not cufilt:
        pytest.skip("cuobjdump / cu++filt not installed: the compiled kernels cannot be listed")
    syms = subprocess.run([cuobjdump, "-symbols", _greedy_native.LIB_PATH], capture_output=True, text=True, check=True).stdout
    mangled = [line.split()[-1] for line in syms.splitlines() if "STO_ENTRY" in line]
    names = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    assert {strip_signature(n) for n in names} == set(GG.KERNELS)
    own = defined_tests("test_gpu_greedy.py")
    for name, tests in GG.KERNELS.items():
        assert tests and set(tests) <= own, (name, tests)


def test_header_and_exports_agree():
    hdr = open(os.path.join(ROOT, "include", "ovc_greedy.h")).read()
    declared = set(re.findall(r"\b(ovc_greedy_[a-z_0-9]+)\s*\(", hdr)) - {"ovc_greedy_layout"}
    assert declared == set(_greedy_native.EXPORTED_SYMBOLS)
    lib = _greedy_native.lib()
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.ovc_greedy_abi_version() == _greedy_native.ABI_VERSION == int(re.search(r"OVC_GREEDY_ABI_VERSION (\d+)", hdr).group(1))


def test_bad_arguments_are_refused():
    """Argument checks run before any launch, so they answer without a device."""
    lib = _greedy_native.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.addressof(buf)
    ok = dict(layouts=p, greedy=p, plans=p, n_layouts=1, state=p, player=p, done=None, prev=p, n_envs=0, state_words=16,
              seed=0, counter=p, actions=p, stream=None)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ovc_greedy_actions(*[a[k] for k in ok]), lib.ovc_greedy_last_error().decode()

    assert call() == (0, call()[1])  # nothing to do for n_envs = 0
    for kw, msg in ((dict(state=None), "null pointer"), (dict(counter=None), "null pointer"), (dict(n_layouts=0), "n_layouts"),
                    (dict(n_layouts=257), "n_layouts"), (dict(n_envs=-1), "negative n_envs"), (dict(state_words=24), "state_words"),
                    (dict(state=p + 4), "aligned"), (dict(counter=p + 4), "aligned"), (dict(prev=p + 2), "aligned")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)


def _env(n=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n)


def test_refused_greedy_configurations():
    """The Boltzmann variants, a greedy learner, a greedy population member of either class."""
    for kw in (dict(hl_boltzmann_rational=True), dict(ll_boltzmann_rational=True), dict(auto_unstuck=False)):
        with pytest.raises(ValueError, match="defaults only"):
            G.GreedyHumanModel(**kw)
    with pytest.raises(AssertionError, match="does not learn"):
        SelfPlayRollout(_env(), model=G.GreedyHumanModel())
    with pytest.raises(AssertionError, match="population member is an RllibShapedCNN or a BCPolicy"):
        AgentPairRollout(_env(), (RllibShapedCNN(5, 4), [BCPolicy(), G.GreedyHumanModel()]))
    with pytest.raises(AssertionError, match="a partner is a BCPolicy, an RllibShapedCNN or a list of them"):
        SelfPlayRollout(_env(), model=RllibShapedCNN(5, 4), partner=[G.GreedyHumanModel()], autocast_dtype=None, fused_first_layer=False)
