"""Live differential tests against the UNMODIFIED reference (skipped unless OVC_REFERENCE names a checkout of it or
oracle/_ref holds the copy build() makes from OVC_REFERENCE_SRC).  Every bundled 2-player layout, fresh random traces each
run of the seed list: the C oracle vs the reference's own get_state_transition / lossless_state_encoding /
featurize_state / potential_function.  This is what keeps the oracle pinned beyond the stored fixtures."""
import json

import numpy as np
import pytest

from oracle import cpu, refboot
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.state import OvercookedState

pytestmark = pytest.mark.reference

ALL_LAYOUTS = []
for _n in L.layout_names():
    try:
        L.compile_layout(_n)
        ALL_LAYOUTS.append(_n)
    except ValueError:
        pass


def _events_mask(ns, infos, agent):
    m = 0
    for i, name in enumerate(ns.mdp.EVENT_TYPES):
        if infos["event_infos"][name][agent]:
            m |= 1 << i
    return m


@pytest.mark.parametrize("name", ALL_LAYOUTS)
def test_layout_against_live_reference(name):
    ns = refboot.boot()
    m = refboot.make_mdp(ns, name)
    _differential(ns, m, L.compile_layout(name), name)


@pytest.mark.parametrize("seed", range(100, 112))
def test_generated_layouts_against_live_reference(seed):
    """LayoutGenerator: the same numpy seed gives the same MDP here and in the reference; then the usual
    differential run (dynamics, encodings, features, potential) on that generated MDP."""
    import copy
    import importlib

    from overcooked_ai_b200 import layout_generator as LG

    ns = refboot.boot()
    ref_lg = importlib.import_module("overcooked_ai_py.mdp.layout_generator")
    variants = [
        ({"inner_shape": (5, 4), "prop_empty": 0.8, "prop_feats": 0.2, "display": False, "recipe_values": [20], "recipe_times": [20],
          "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}]}, (5, 4)),
        ({"inner_shape": (6, 5), "prop_empty": 0.5, "prop_feats": 0.3, "display": False, "feature_types": ["P", "D", "S", "O", "T"],
          "start_all_orders": [{"ingredients": ["onion", "tomato"]}, {"ingredients": ["onion", "onion", "onion"]}],
          "start_bonus_orders": [{"ingredients": ["onion", "tomato"]}]}, (7, 6)),
        ({"inner_shape": (7, 5), "prop_empty": 0.6, "prop_feats": 0.4, "display": False,
          "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}]}, (9, 6)),
    ]
    params, outer = variants[seed % len(variants)]
    np.random.seed(seed)
    m = ref_lg.LayoutGenerator(ref_lg.MDPParamsGenerator.from_fixed_param(copy.deepcopy(params)), outer_shape=outer).generate_padded_mdp()
    np.random.seed(seed)
    try:
        mine = LG.LayoutGenerator(LG.MDPParamsGenerator.from_fixed_param(copy.deepcopy(params)), outer_shape=outer).generate_padded_mdp()
    except ValueError:
        assert len(m.get_pot_locations()) > 4  # the only rejection: more pots than the record format holds
        return
    assert ["".join(r) for r in mine.terrain_mtx] == ["".join(r) for r in m.terrain_mtx]
    assert [tuple(p) for p in mine.start_player_positions] == [tuple(p) for p in m.start_player_positions]
    key = lambda orders: sorted(tuple(sorted(o["ingredients"])) for o in orders)
    assert key(mine.start_all_orders) == key(m.start_all_orders) and key(mine.start_bonus_orders) == key(m.start_bonus_orders)
    _differential(ns, m, mine.compiled, "generated-%d" % seed)


def _differential(ns, m, cl, name):
    refboot.use_mdp(ns, m)
    tab, starts, S = L.build_tables([cl])
    small = cl.width * cl.height <= 50
    if small:
        holder = refboot.LitePlannerHolder(ns, m)
        lut = cl.feature_lut().view(np.uint8).reshape(1, -1)
        pt, cst, gpow = L.build_potential_tables([cl], 0.99)
    # OVC_FUZZ_EPISODES / OVC_FUZZ_STEPS / OVC_FUZZ_SEED scale this into a fuzzing campaign (defaults: 6 x 60, seed 0)
    import os

    episodes, steps = int(os.environ.get("OVC_FUZZ_EPISODES", "6")), int(os.environ.get("OVC_FUZZ_STEPS", "60"))
    seed = sum(map(ord, name)) + int(os.environ.get("OVC_FUZZ_SEED", "0"))
    np.random.seed(seed)
    rng = np.random.RandomState(seed)
    fn = m.get_random_start_state_fn(random_start_pos=True, rnd_obj_prob_thresh=0.6)
    n_obs = 0
    for ep in range(episodes):
        st = fn() if ep else m.get_standard_start_state()
        for t in range(steps):
            a = rng.randint(0, 6, size=2)
            if rng.rand() < 0.4:
                a[rng.randint(2)] = 5
            rec = L.pack_state(cl, OvercookedState.from_dict(st.to_dict()), 0, S)[None].copy()
            if t % 10 == 0:
                enc = cpu.encode_lossless(tab, rec, cl.width, cl.height, 400)[0]
                assert np.array_equal(enc, np.stack(m.lossless_state_encoding(st, horizon=400))), (name, ep, t)
                if small:
                    f = cpu.featurize(tab, lut, rec, 2)[0]
                    assert np.array_equal(f, np.stack(m.featurize_state(st, holder, num_pots=2))), (name, ep, t)
                    phi = cpu.potential(tab, pt, cst, gpow, rec)[0]
                    assert phi == m.potential_function(st, holder.motion_planner, gamma=0.99), (name, ep, t)
                n_obs += 1
            ja = tuple(ns.actions.Action.INDEX_TO_ACTION[int(x)] for x in a)
            st, infos = m.get_state_transition(st, ja)
            sp, sh, dn, ev = cpu.step(tab, starts, rec, a[None].astype(np.int32), horizon=0)
            want = L.pack_state(cl, OvercookedState.from_dict(st.to_dict()), 0, S)
            assert np.array_equal(rec[0], want), (name, ep, t, ja)
            assert sp[0] == sum(infos["sparse_reward_by_agent"]) and sh[0].tolist() == list(infos["shaped_reward_by_agent"])
            assert [int(ev[0, 0]) & 0x1FFFFFF, int(ev[0, 1]) & 0x1FFFFFF] == [_events_mask(ns, infos, 0), _events_mask(ns, infos, 1)]
    assert n_obs == episodes * ((steps + 9) // 10)


def _random_mdp_params(rng):
    """A random, valid set of MDP parameter overrides (orders, bonus orders, recipe values / times by any of the
    reference's three mechanisms, order bonus, shaping rewards, old dynamics)."""
    onion, tomato = "onion", "tomato"
    recipes = [[onion], [tomato], [onion, onion], [onion, tomato], [tomato, tomato], [onion] * 3, [onion, onion, tomato],
               [onion, tomato, tomato], [tomato] * 3]
    p = {}
    old = rng.rand() < 0.25
    pool = [r for r in recipes if len(r) == 3] if old else recipes
    k = rng.randint(1, len(pool) + 1)
    orders = [pool[i] for i in sorted(rng.choice(len(pool), k, replace=False))]
    p["start_all_orders"] = [{"ingredients": list(r)} for r in orders]
    p["start_bonus_orders"] = []  # always overridden: a layout's own bonus orders need not be among the new orders
    if rng.rand() < 0.5:
        nb = rng.randint(1, len(orders) + 1)
        p["start_bonus_orders"] = [{"ingredients": list(orders[i])} for i in sorted(rng.choice(len(orders), nb, replace=False))]
        p["order_bonus"] = int(rng.choice([2, 3, 5]))
    mech = rng.randint(4)
    if mech == 0:
        p["recipe_values"] = [int(v) for v in rng.randint(1, 60, size=len(orders))]
        p["recipe_times"] = [int(v) for v in rng.randint(1, 30, size=len(orders))]
    elif mech == 1:
        p["onion_value"], p["tomato_value"] = int(rng.randint(1, 25)), int(rng.randint(1, 25))
        p["onion_time"], p["tomato_time"] = int(rng.randint(1, 12)), int(rng.randint(1, 12))
    elif mech == 2:
        p["delivery_reward"], p["cook_time"] = int(rng.randint(1, 50)), int(rng.randint(1, 25))
    if rng.rand() < 0.5:
        p["rew_shaping_params"] = {"PLACEMENT_IN_POT_REW": int(rng.randint(0, 9)), "DISH_PICKUP_REWARD": int(rng.randint(0, 9)),
                                   "SOUP_PICKUP_REWARD": int(rng.randint(0, 9)), "DISH_DISP_DISTANCE_REW": 0,
                                   "POT_DISTANCE_REW": 0, "SOUP_DISTANCE_REW": 0}
    if old:
        p["old_dynamics"] = True
    return p


@pytest.mark.parametrize("seed", range(16))
def test_random_mdp_parameters_against_live_reference(seed):
    """Parameter overrides of from_layout_name (overcooked_mdp.py:1090-1172: orders, bonus orders, the three ways to
    set recipe values / times, order bonus, shaping rewards, old dynamics): same differential run as above."""
    import copy

    ns = refboot.boot()
    rng = np.random.RandomState(1000 + seed)
    name = ["cramped_room", "counter_circuit", "asymmetric_advantages", "cramped_room_tomato"][seed % 4]
    if name not in ALL_LAYOUTS:
        name = "cramped_room"
    params = _random_mdp_params(rng)
    try:
        m = refboot.make_mdp(ns, name, **copy.deepcopy(params))
    except ValueError:  # e.g. a scalar override on a layout that prices recipes per ingredient: same verdict here
        with pytest.raises(ValueError):
            L.compile_layout(name, **copy.deepcopy(params))
        return
    cl = L.compile_layout(name, **copy.deepcopy(params))
    _differential(ns, m, cl, "%s-params-%d" % (name, seed))


def test_recipe_config_conflicts_raise_like_the_reference():
    """Recipe.configure's validity rules (overcooked_mdp.py:236-300) on every pair of mechanisms."""
    ns = refboot.boot()
    orders = [{"ingredients": ["onion", "onion", "onion"]}]
    cases = [
        {"onion_value": 3}, {"tomato_time": 4}, {"onion_value": 3, "tomato_value": 2, "delivery_reward": 9},
        {"onion_value": 3, "tomato_value": 2, "recipe_values": [5], "start_all_orders": orders},
        {"recipe_values": [5], "delivery_reward": 9, "start_all_orders": orders},
        {"onion_time": 3, "tomato_time": 2, "cook_time": 9},
        {"onion_time": 3, "tomato_time": 2, "recipe_times": [5], "start_all_orders": orders},
        {"recipe_times": [5], "cook_time": 9, "start_all_orders": orders},
        {"recipe_values": [5]}, {"recipe_times": [5, 6], "start_all_orders": orders},
        {"recipe_values": [5], "recipe_times": [7], "start_all_orders": orders},  # valid
        {"onion_value": 3, "tomato_value": 2, "onion_time": 4, "tomato_time": 5},  # valid
    ]
    for kw in cases:
        import copy

        try:
            refboot.make_mdp(ns, "cramped_room", **copy.deepcopy(kw))
            ok = True
        except ValueError:
            ok = False
        if ok:
            L.compile_layout("cramped_room", **copy.deepcopy(kw))
        else:
            with pytest.raises(ValueError):
                L.compile_layout("cramped_room", **copy.deepcopy(kw))


def test_grid_validity_rules_against_live_reference():
    """Same grids, same verdict and message as OvercookedGridworld.from_grid (overcooked_mdp.py:1175-1187, 2064-2115)."""
    from overcooked_ai_b200.mdp import OvercookedGridworld

    ns = refboot.boot()
    grids = [
        ["XXPXX", "O  2O", "X1  X", "XDXSX"], ["XXPXX", "O  2", "X1  X", "XDXSX"], ["XXPXX", "   2O", "X1  X", "XDXSX"],
        ["XXPXX", "O  2 ", "X1  X", "XDXSX"], ["XX XX", "O  2O", "X1  X", "XDXSX"], ["XXPXX", "O  2O", "X1  X", "XD1SX"],
        ["XXPXX", "O   O", "X   X", "XDXSX"], ["XXPXX", "O  3O", "X1  X", "XDXSX"], ["XXPXX", "O ?2O", "X1  X", "XDXSX"],
        ["XXPXX", "O  2O", "X1  X", "XXXSX"], ["XXPXX", "O  2O", "X1  X", "XDXXX"], ["XXXXX", "O  2O", "X1  X", "XDXSX"],
        ["XXPXX", "X  2X", "X1  X", "XDXSX"], ["XTPXX", "X  2X", "X1  X", "XDXSX"],
    ]
    for g in grids:
        try:
            ns.mdp.OvercookedGridworld.from_grid(g)
            want = None
        except AssertionError as e:
            want = str(e)
        try:
            OvercookedGridworld.from_grid(g)
            got = None
        except AssertionError as e:
            got = str(e)
        assert got == want, (g, got, want)


@pytest.mark.parametrize("name", ["cramped_room", "counter_circuit", "asymmetric_advantages", "forced_coordination_tomato"])
def test_host_random_start_states_against_live_reference(name):
    """get_random_start_state_fn (overcooked_mdp.py:1307-1369) of the drop-in mdp: same numpy seed, same states."""
    from overcooked_ai_b200.mdp import OvercookedGridworld

    if name not in ALL_LAYOUTS:
        pytest.skip("layout not bundled")
    ns = refboot.boot()
    m = refboot.make_mdp(ns, name)
    mine = OvercookedGridworld.from_layout_name(name)
    assert mine.get_valid_joint_player_positions() == m.get_valid_joint_player_positions()
    for pos, thr in ((True, 0.0), (False, 0.7), (True, 0.5), (True, 1.0)):
        for seed in range(6):
            refboot.use_mdp(ns, m)
            np.random.seed(seed)
            f = m.get_random_start_state_fn(random_start_pos=pos, rnd_obj_prob_thresh=thr)
            want = [json.loads(json.dumps(f().to_dict())) for _ in range(4)]
            np.random.seed(seed)
            g = mine.get_random_start_state_fn(random_start_pos=pos, rnd_obj_prob_thresh=thr)
            got = [json.loads(json.dumps(g().to_dict())) for _ in range(4)]
            for a, b in zip(got, want):
                a["objects"].sort(key=lambda o: o["position"]), b["objects"].sort(key=lambda o: o["position"])
                assert a == b, (name, pos, thr, seed)
            st = g()
            assert dict(mine.get_pot_states(st)) == dict(m.get_pot_states(ns.mdp.OvercookedState.from_dict(json.loads(json.dumps(st.to_dict())))))


def test_call_signatures_of_the_boundary_match_the_reference():
    """SURVEY 8b: the drop-in classes keep the reference's parameter names, order and kinds on every entry point of
    the path (extra trailing parameters — ``device``, ``**kwargs`` — are allowed), and its simple default values."""
    import inspect

    from overcooked_ai_b200 import env as E
    from overcooked_ai_b200 import mdp as M

    ns = refboot.boot()
    env_names = ["__init__", "from_mdp", "step", "reset", "is_done", "potential", "lossless_state_encoding_mdp",
                 "featurize_state_mdp", "execute_plan"]
    mdp_names = ["from_layout_name", "from_grid", "get_state_transition", "lossless_state_encoding", "featurize_state",
                 "potential_function", "get_random_start_state_fn", "get_standard_start_state", "get_pot_states", "get_actions",
                 "get_valid_joint_player_positions", "get_valid_player_positions", "get_pot_locations",
                 "get_counter_locations", "get_serving_locations", "get_dish_dispenser_locations",
                 "get_onion_dispenser_locations", "get_tomato_dispenser_locations", "get_terrain_type_at_pos", "is_terminal"]
    pairs = [(getattr(ns.env.OvercookedEnv, n), getattr(E.OvercookedEnv, n)) for n in env_names]
    pairs += [(getattr(ns.env.Overcooked, n), getattr(E.Overcooked, n)) for n in ("step", "reset")]
    pairs += [(getattr(ns.mdp.OvercookedGridworld, n), getattr(M.OvercookedGridworld, n)) for n in mdp_names]
    for ref_fn, my_fn in pairs:
        ref_p = list(inspect.signature(ref_fn).parameters.values())
        my_p = list(inspect.signature(my_fn).parameters.values())
        assert [(p.name, p.kind) for p in my_p[:len(ref_p)]] == [(p.name, p.kind) for p in ref_p], ref_fn.__qualname__
        for a, b in zip(ref_p, my_p):
            if isinstance(a.default, (int, float, bool, str, type(None))) and a.default is not inspect.Parameter.empty:
                assert a.default == b.default, (ref_fn.__qualname__, a.name, a.default, b.default)
