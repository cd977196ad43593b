#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference (needs OVC_REFERENCE=<a checkout of it>).

Every array written here comes out of the reference's own Python functions
(OvercookedGridworld.get_state_transition / lossless_state_encoding / featurize_state, imported
from the checkout through oracle/refboot.py); the reference's own golden vectors
(src/overcooked_ai_py/data/testing/...) are replayed and asserted on the way, so the fixtures pin
"reference as run here == reference's published expectations".  States are stored as packed int32
records (include/ovc_b200.h) produced by overcooked_ai_b200.layout.pack_state from the reference
state's ``to_dict()``; a JSON sample of raw ``to_dict()`` output is stored next to them so the
packing itself is checked too.

Run:  python tools/make_golden.py          (about two minutes; rewrites tests/golden/)
"""
import json
import os
import pickle
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

from oracle import refboot  # noqa: E402
from overcooked_ai_b200 import layout as L  # noqa: E402
from overcooked_ai_b200.state import OvercookedState  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
TESTING = os.path.join(refboot.REFERENCE_ROOT, "src", "overcooked_ai_py", "data", "testing")


def events_mask(ns, infos, agent):
    m = 0
    for i, name in enumerate(ns.mdp.EVENT_TYPES):
        if infos["event_infos"][name][agent]:
            m |= 1 << i
    return m


def jsonable(d):
    return json.loads(json.dumps(d))


def pack_ref(cl, ref_state, S):
    return L.pack_state(cl, OvercookedState.from_dict(ref_state.to_dict()), 0, S)


def run_trace(ns, m, cl, start_state, actions, S, obs_every=0, mlam=None, horizon=400):
    """Reference get_state_transition along one action sequence.  Returns per-step arrays."""
    st = start_state
    T = len(actions)
    states = np.zeros((T + 1, S), np.int32)
    sparse = np.zeros((T, 2), np.int32)
    shaped = np.zeros((T, 2), np.int32)
    events = np.zeros((T, 2), np.int32)
    states[0] = pack_ref(cl, st, S)
    for t in range(T):
        ja = tuple(ns.actions.Action.INDEX_TO_ACTION[a] for a in actions[t])
        st, infos = m.get_state_transition(st, ja)
        states[t + 1] = pack_ref(cl, st, S)
        sparse[t] = infos["sparse_reward_by_agent"]
        shaped[t] = infos["shaped_reward_by_agent"]
        events[t] = [events_mask(ns, infos, 0), events_mask(ns, infos, 1)]
    return states, sparse, shaped, events, st


def biased_actions(rng, T, p_interact):
    a = rng.randint(0, 5, size=(T, 2))
    a[rng.rand(T, 2) < p_interact] = 5
    return a.astype(np.int32)


def gen_dynamics_mdp_test(ns):
    """The reference's golden trajectory (testing/overcooked_test.py:516-525, expected.json)."""
    with open(os.path.join(TESTING, "test_mdp_dynamics", "expected.json")) as f:
        traj = json.load(f)
    mdp_params = traj["mdp_params"][0]
    m = ns.mdp.OvercookedGridworld.from_layout_name(**mdp_params) if "layout_name" in mdp_params and len(mdp_params) == 1 else refboot.make_mdp(ns, "mdp_test")
    refboot.use_mdp(ns, m)
    cl = L.compile_layout("mdp_test")
    S = cl.state_words
    states = [ns.mdp.OvercookedState.from_dict(s) for s in traj["ep_states"][0]]
    act_idx = []
    for ja in traj["ep_actions"][0]:
        ja = tuple(tuple(a) if isinstance(a, list) else a for a in ja)
        act_idx.append([ns.actions.Action.ACTION_TO_INDEX[a] for a in ja])
    act_idx = np.array(act_idx, np.int32)
    rewards = np.array(traj["ep_rewards"][0], np.int64)
    T = len(act_idx)
    packed, sparse, shaped, events, _ = run_trace(ns, m, cl, states[0], act_idx, S)
    mism = 0
    for t in range(T - 1):  # the reference's own expected next states and rewards
        mism += int(not np.array_equal(packed[t + 1], pack_ref(cl, states[t + 1], S)))
        mism += int(sparse[t].sum() != rewards[t])
    assert mism == 0, "reference-as-run-here diverges from its own golden trajectory"
    sample = {str(t): jsonable(states[t].to_dict()) for t in range(0, T, 97)}
    np.savez_compressed(
        os.path.join(GOLD, "dynamics_mdp_test.npz"), layout="mdp_test", horizon=1500, actions=act_idx,
        states=packed, sparse=sparse, shaped=shaped, events=events, to_dict_sample=json.dumps(sample),
    )
    print("dynamics_mdp_test: %d transitions, deliveries=%d, sum sparse=%d" % (T, int((sparse.sum(1) > 0).sum()), int(sparse.sum())))


TRACE_LAYOUTS = [
    # (fixture name, layout, params, episodes, steps)
    ("cramped_room", "cramped_room", {}, 96, 120),
    ("asymmetric_advantages", "asymmetric_advantages", {}, 48, 120),
    ("coordination_ring", "coordination_ring", {}, 48, 120),
    ("forced_coordination", "forced_coordination", {}, 48, 120),
    ("counter_circuit", "counter_circuit", {}, 96, 120),
    ("mdp_test", "mdp_test", {}, 128, 120),
    ("bonus_order_test", "bonus_order_test", {}, 64, 100),
    ("cramped_room_tomato", "cramped_room_tomato", {}, 64, 100),
    ("forced_coordination_tomato", "forced_coordination_tomato", {}, 32, 100),
    ("cramped_room_old_dynamics", "cramped_room", {"old_dynamics": True}, 48, 120),
    ("marshmallow_experiment", "marshmallow_experiment", {}, 24, 100),
    ("corridor", "corridor", {}, 8, 100),
    ("tutorial_1", "tutorial_1", {}, 12, 100),
]


def gen_traces(ns, name, layout, params, episodes, steps, seed):
    m = refboot.make_mdp(ns, layout, **params)
    refboot.use_mdp(ns, m)
    cl = L.compile_layout(layout, **params)
    S = cl.state_words
    rng = np.random.RandomState(seed)
    np.random.seed(seed)
    fn_std = m.get_standard_start_state
    fn_rnd = m.get_random_start_state_fn(random_start_pos=True, rnd_obj_prob_thresh=0.6)
    all_states, all_actions, all_sparse, all_shaped, all_events = [], [], [], [], []
    sample = {}
    holder = refboot.LitePlannerHolder(ns, m)
    obs_states, obs_lossless, obs_feat = [], [], {0: [], 1: [], 2: [], 3: []}
    for ep in range(episodes):
        if ep % 4 == 0:
            start = fn_std()
        else:
            start = fn_rnd()
            if ep % 4 == 2:
                start.timestep = 400 - steps + 10  # exercises the urgency plane and the horizon edge
        acts = biased_actions(rng, steps, [0.17, 0.3, 0.45][ep % 3])
        states, sparse, shaped, events, _ = run_trace(ns, m, cl, start, acts, S)
        all_states.append(states), all_actions.append(acts), all_sparse.append(sparse)
        all_shaped.append(shaped), all_events.append(events)
        if ep < 3:
            sample["%d:0" % ep] = jsonable(start.to_dict())
        # observations on a subsample of the visited states, straight from the reference
        for t in range(0, steps + 1, 7):
            st = L.unpack_state(cl, states[t])
            ref_st = ns.mdp.OvercookedState.from_dict(jsonable(st.to_dict()))
            enc = m.lossless_state_encoding(ref_st, horizon=400)
            obs_states.append(states[t])
            obs_lossless.append(np.stack(enc).astype(np.int16))
            for npots in obs_feat:
                obs_feat[npots].append(np.stack(m.featurize_state(ref_st, holder, num_pots=npots)))
    ev = np.concatenate(all_events).reshape(-1)
    cover = [int(((ev >> i) & 1).sum()) for i in range(25)]
    out = dict(
        layout=layout, params=json.dumps(params), horizon=400,
        states=np.stack(all_states), actions=np.stack(all_actions), sparse=np.stack(all_sparse),
        shaped=np.stack(all_shaped), events=np.stack(all_events), to_dict_sample=json.dumps(sample),
        obs_states=np.stack(obs_states), obs_lossless=np.stack(obs_lossless),
    )
    for npots, v in obs_feat.items():
        arr = np.stack(v)
        assert np.array_equal(arr, arr.astype(np.int16)), "featurize_state values are small integers"
        out["obs_feat_%d" % npots] = arr.astype(np.int16)
    np.savez_compressed(os.path.join(GOLD, "trace_%s.npz" % name), **out)
    print("trace_%s: %d eps x %d steps, S=%d, sparse sum=%d, event coverage=%s" % (
        name, episodes, steps, S, int(np.stack(all_sparse).sum()), cover))


def philox4x32_10(key, c0, c1, c2, c3):
    """Philox4x32-10 (the generator of include/ovc_b200.h's random start states), plain Python integers."""
    k0, k1 = key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c3 ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


def config1_actions(seed, T=400, env_id=0):
    """BASELINE config 1 / SURVEY 8d: a[t, agent] uniform in 0..5 from a counter-based generator keyed by the seed,
    counter (env id, t): word `agent` of the block, scaled by multiply-high."""
    a = np.zeros((T, 2), np.int32)
    for t in range(T):
        v = philox4x32_10(seed, env_id, t, 0, 0)
        a[t] = [(v[0] * 6) >> 32, (v[1] * 6) >> 32]
    return a


def gen_config1(ns):
    """BASELINE config 1: cramped_room, ONE environment, horizon 400, standard start state, uniform random joint actions
    (seeds 0..7), stepped through the reference's OvercookedEnv: every state / reward / event flag, and the episode
    info the env hands out with the last transition."""
    m = refboot.make_mdp(ns, "cramped_room")
    refboot.use_mdp(ns, m)
    cl = L.compile_layout("cramped_room")
    S, T = cl.state_words, 400
    holder = refboot.LitePlannerHolder(ns, m)
    states, actions, sparse, shaped, events, infos_out = [], [], [], [], [], []
    obs_states, obs_lossless, obs_feat = [], [], {0: [], 1: [], 2: [], 3: []}
    sample = {}
    for seed in range(8):
        env = refboot.make_env(ns, m, horizon=T)
        env._mp = object()
        acts = config1_actions(seed, T)
        st_arr = np.zeros((T + 1, S), np.int32)
        sp, sh, ev = np.zeros((T, 2), np.int32), np.zeros((T, 2), np.int32), np.zeros((T, 2), np.int32)
        st_arr[0] = pack_ref(cl, env.state, S)
        for t in range(T):
            ja = tuple(ns.actions.Action.INDEX_TO_ACTION[int(a)] for a in acts[t])
            prev = env.state
            _, mdp_infos = m.get_state_transition(prev, ja)  # for the event flags (the env keeps only their timesteps)
            nxt, r, done, info = env.step(ja)
            st_arr[t + 1] = pack_ref(cl, nxt, S)
            sp[t], sh[t] = info["sparse_r_by_agent"], info["shaped_r_by_agent"]
            ev[t] = [events_mask(ns, mdp_infos, 0), events_mask(ns, mdp_infos, 1)]
            assert r == sum(info["sparse_r_by_agent"]) and done == (t == T - 1)
            if seed < 3 and t in (0, 150, 399):
                sample["%d:%d" % (seed, t)] = jsonable(prev.to_dict())
            if t % 25 == 0:
                obs_states.append(st_arr[t])
                obs_lossless.append(np.stack(m.lossless_state_encoding(prev, horizon=T)).astype(np.int16))
                for npots in obs_feat:
                    obs_feat[npots].append(np.stack(m.featurize_state(prev, holder, num_pots=npots)))
        ep = info["episode"]
        infos_out.append({
            "ep_sparse_r": int(ep["ep_sparse_r"]), "ep_shaped_r": int(ep["ep_shaped_r"]),
            "ep_sparse_r_by_agent": [int(v) for v in ep["ep_sparse_r_by_agent"]],
            "ep_shaped_r_by_agent": [int(v) for v in ep["ep_shaped_r_by_agent"]], "ep_length": int(ep["ep_length"]),
            "game_stats": {k: [[int(x) for x in lst] for lst in v] for k, v in ep["ep_game_stats"].items()
                           if k in ns.mdp.EVENT_TYPES},
        })
        states.append(st_arr), actions.append(acts), sparse.append(sp), shaped.append(sh), events.append(ev)
    out = dict(layout="cramped_room", params=json.dumps({}), horizon=T, states=np.stack(states), actions=np.stack(actions),
               sparse=np.stack(sparse), shaped=np.stack(shaped), events=np.stack(events), to_dict_sample=json.dumps(sample),
               obs_states=np.stack(obs_states), obs_lossless=np.stack(obs_lossless), episode_info=json.dumps(infos_out))
    for npots, v in obs_feat.items():
        out["obs_feat_%d" % npots] = np.stack(v).astype(np.int16)
    np.savez_compressed(os.path.join(GOLD, "trace_config1_cramped_room.npz"), **out)
    print("trace_config1_cramped_room: 8 seeds x %d steps, shaped sums %s, sparse sums %s" % (
        T, [i["ep_shaped_r"] for i in infos_out], [i["ep_sparse_r"] for i in infos_out]))


def gen_greedy_cramped_room(ns):
    """The reference's featurisation goldens (testing/overcooked_test.py:1005-1093): 5 seeded
    GreedyHumanModel self-play games on cramped_room; expected.pickle / expected_{0,1,2}.pickle."""
    m = refboot.make_mdp(ns, "cramped_room")
    refboot.use_mdp(ns, m)
    cl = L.compile_layout("cramped_room")
    S = cl.state_words
    mlam = ns.planners.MediumLevelActionManager.from_pickle_or_compute(m, ns.planners.NO_COUNTERS_PARAMS, force_compute=True)
    env = ns.env.OvercookedEnv.from_mdp(m, horizon=400, info_level=0)
    env._mp = mlam.motion_planner
    pair = ns.agent.AgentPair(ns.agent.GreedyHumanModel(mlam), ns.agent.GreedyHumanModel(mlam))
    np.random.seed(0)
    trajs = env.get_rollouts(pair, num_games=5, info=False)
    with open(os.path.join(TESTING, "test_lossless_state_featurization", "expected.pickle"), "rb") as f:
        exp_lossless = np.array(pickle.load(f))
    got = np.array([[m.lossless_state_encoding(s) for s in ep] for ep in trajs["ep_states"]])
    assert np.array_equal(exp_lossless, got), "lossless golden not reproduced"
    feats = {}
    for npots in range(3):
        with open(os.path.join(TESTING, "test_state_featurization", "expected_%d.pickle" % npots), "rb") as f:
            exp = np.array(pickle.load(f))
        got_f = np.array([[m.featurize_state(s, mlam, num_pots=npots) for s in ep] for ep in trajs["ep_states"]])
        assert np.array_equal(exp, got_f), "featurize golden %d not reproduced" % npots
        assert np.array_equal(exp, exp.astype(np.int16))
        feats[npots] = exp.astype(np.int16)
    states = np.array([[pack_ref(cl, s, S) for s in ep] for ep in trajs["ep_states"]], np.int32)
    actions = np.array(
        [[[ns.actions.Action.ACTION_TO_INDEX[a] for a in ja] for ja in ep] for ep in trajs["ep_actions"]], np.int32
    )
    rewards = np.array(trajs["ep_rewards"]).astype(np.int32)
    # replay through get_state_transition to also record shaped rewards and events
    sparse, shaped, events = [], [], []
    for e in range(states.shape[0]):
        st, sp, sh, ev, _ = run_trace(ns, m, cl, trajs["ep_states"][e][0], actions[e], S)
        assert np.array_equal(st[:-1], states[e]) and np.array_equal(sp.sum(1), rewards[e])
        sparse.append(sp), shaped.append(sh), events.append(ev)
    np.savez_compressed(
        os.path.join(GOLD, "greedy_cramped_room.npz"), layout="cramped_room", horizon=400,
        states=states, actions=actions, sparse=np.stack(sparse), shaped=np.stack(shaped), events=np.stack(events),
        lossless=exp_lossless.astype(np.uint8), feat_0=feats[0], feat_1=feats[1], feat_2=feats[2],
    )
    print("greedy_cramped_room: states %s, ep returns %s" % (states.shape, rewards.sum(1).tolist()))


def gen_planner_luts(ns):
    """min_cost_to_feature argmins of the reference MotionPlanner for every bundled 2-player layout,
    in the engine's LUT form — pins CompiledLayout.feature_lut()."""
    out = {}
    for name in L.layout_names():
        try:
            cl = L.compile_layout(name)
        except ValueError:
            continue
        if cl.width * cl.height > 70:  # corridor etc.: the reference planner needs minutes; covered by trace_corridor
            continue
        m = refboot.make_mdp(ns, name)
        refboot.use_mdp(ns, m)
        mp = ns.planners.MotionPlanner(m)
        lut = np.zeros((256, 4), L.FEAT_LUT_DTYPE)
        lut["pot_order"] = L.NO_SLOT
        for pos in m.get_valid_player_positions():
            for oi, o in enumerate(ns.actions.Direction.ALL_DIRECTIONS):
                e = lut[L.pos_byte(pos), oi]
                for key, locs in (("d_onion", m.get_onion_dispenser_locations()), ("d_tomato", m.get_tomato_dispenser_locations()),
                                  ("d_dish", m.get_dish_dispenser_locations()), ("d_serve", m.get_serving_locations())):
                    _, f = mp.min_cost_to_feature((pos, o), locs, with_argmin=True)
                    if f is not None:
                        e[key] = (f[0] - pos[0], f[1] - pos[1])
                pots = m.get_pot_locations().copy()
                for k in range(len(pots)):
                    _, f = mp.min_cost_to_feature((pos, o), pots, with_argmin=True)
                    if f is None:
                        break
                    e["pot_order"][k] = cl.slot_of[f]
                    pots.remove(f)
        out[name] = lut.view(np.uint8).reshape(-1)
    np.savez_compressed(os.path.join(GOLD, "planner_luts.npz"), **out)
    print("planner_luts: %d layouts" % len(out))


def gen_human_2020(ns):
    """Real human-human games (src/human_aware_rl/static/human_data/dummy/dummy_2020_hh_trials.csv; the
    reference replays such data in human_aware_rl/human/tests.py:197-211): every recorded transition is
    pushed through the reference's get_state_transition and must land on the next recorded state and
    reward; stored in the trace-fixture format."""
    import pandas as pd

    csv = os.path.join(refboot.REFERENCE_ROOT, "src", "human_aware_rl", "static", "human_data", "dummy", "dummy_2020_hh_trials.csv")
    df = pd.read_csv(csv)
    for (layout, trial), g in df.groupby(["layout_name", "trial_id"], sort=False):
        m = refboot.make_mdp(ns, layout)
        refboot.use_mdp(ns, m)
        cl = L.compile_layout(layout)
        S = cl.state_words
        rows = list(g.sort_values("cur_gameloop").itertuples())
        acts = []
        for r in rows:
            ja = [tuple(x) if isinstance(x, list) else x.lower() for x in json.loads(r.joint_action)]
            acts.append([ns.actions.Action.ACTION_TO_INDEX[a] for a in ja])
        acts = np.array(acts, np.int32)
        start = ns.mdp.OvercookedState.from_dict(json.loads(rows[0].state))
        states, sparse, shaped, events, _ = run_trace(ns, m, cl, start, acts, S)
        for t in range(len(rows) - 1):
            exp = ns.mdp.OvercookedState.from_dict(json.loads(rows[t + 1].state))
            assert np.array_equal(states[t + 1], pack_ref(cl, exp, S)), (layout, t)
            assert sparse[t].sum() == rows[t].reward, (layout, t)
        holder = refboot.LitePlannerHolder(ns, m)
        obs_states, obs_lossless, obs_feat = [], [], {0: [], 1: [], 2: [], 3: []}
        for t in range(0, len(rows), 9):
            st = L.unpack_state(cl, states[t])
            ref_st = ns.mdp.OvercookedState.from_dict(jsonable(st.to_dict()))
            obs_states.append(states[t])
            obs_lossless.append(np.stack(m.lossless_state_encoding(ref_st, horizon=400)).astype(np.int16))
            for npots in obs_feat:
                obs_feat[npots].append(np.stack(m.featurize_state(ref_st, holder, num_pots=npots)))
        out = dict(layout=layout, params=json.dumps({}), horizon=400, states=states[None], actions=acts[None],
                   sparse=sparse[None], shaped=shaped[None], events=events[None],
                   to_dict_sample=json.dumps({"0": json.loads(rows[0].state), "200": json.loads(rows[200].state)}),
                   obs_states=np.stack(obs_states), obs_lossless=np.stack(obs_lossless))
        for npots, v in obs_feat.items():
            out["obs_feat_%d" % npots] = np.stack(v).astype(np.int16)
        np.savez_compressed(os.path.join(GOLD, "trace_human2020_%s.npz" % layout), **out)
        print("trace_human2020_%s: %d recorded transitions, sparse sum %d, deliveries %d" % (
            layout, len(rows), int(sparse.sum()), int(((events >> 15) & 1).sum())))


def gen_potential(ns):
    """potential_function (overcooked_mdp.py:2920-3250, gamma 0.99 and 0.9) of the reference on the observation
    states of every trace fixture, plus the MotionPlanner costs it consumes — pins the potential oracle/kernel."""
    out = {}
    import glob

    cases = [(n, l, p) for n, l, p, _, _ in TRACE_LAYOUTS]
    for path in sorted(glob.glob(os.path.join(GOLD, "trace_human2020_*.npz"))):
        nm = os.path.basename(path)[len("trace_"):-4]
        cases.append((nm, nm[len("human2020_"):], {}))
    for name, layout, params in cases:
        d = np.load(os.path.join(GOLD, "trace_%s.npz" % name))
        m = refboot.make_mdp(ns, layout, **params)
        refboot.use_mdp(ns, m)
        cl = L.compile_layout(layout, **params)
        if cl.width * cl.height > 70:
            continue  # corridor: the reference planner needs minutes
        mp = ns.planners.MotionPlanner(m)
        states = d["obs_states"]
        phis = np.zeros((len(states), 2), np.float64)
        for k, rec in enumerate(states):
            st = L.unpack_state(cl, rec)
            ref_st = ns.mdp.OvercookedState.from_dict(jsonable(st.to_dict()))
            phis[k, 0] = m.potential_function(ref_st, mp, gamma=0.99)
            phis[k, 1] = m.potential_function(ref_st, mp, gamma=0.9)
        cost = np.full((256, 4, 5), 255, np.int32)
        for pos in m.get_valid_player_positions():
            for oi, o in enumerate(ns.actions.Direction.ALL_DIRECTIONS):
                c = mp.min_cost_to_feature((pos, o), m.get_serving_locations())
                cost[L.pos_byte(pos), oi, 0] = 255 if c == np.inf else int(c)
                for j, pot in enumerate(m.get_pot_locations()):
                    c = mp.min_cost_to_feature((pos, o), [pot])
                    cost[L.pos_byte(pos), oi, 1 + j] = 255 if c == np.inf else int(c)
        out[name + "__phi"] = phis
        out[name + "__cost"] = cost.astype(np.uint8)
        print("potential %s: %d states, phi range [%.3f, %.3f]" % (name, len(states), phis[:, 0].min(), phis[:, 0].max()))
    np.savez_compressed(os.path.join(GOLD, "potential.npz"), **out)


# (name, mdp_gen_params, outer_shape, seeds): the cases of tests/golden/layout_generator.npz
LAYOUTGEN_CASES = [
    ("default", {"inner_shape": (5, 4), "prop_empty": 0.95, "prop_feats": 0.1,
                 "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}], "recipe_values": [20],
                 "recipe_times": [20], "display": False}, (5, 4), range(12)),
    ("ref_test_5x4", {"inner_shape": (5, 4), "prop_empty": 0.8, "prop_feats": 0.2,
                      "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}], "recipe_values": [20],
                      "recipe_times": [20], "display": False}, (5, 4), range(12)),  # overcooked_test.py:1318-1331
    ("ref_test_6x5_tomato", {"prop_feats": 0.9, "feature_types": ["P", "D", "S", "O", "T"], "prop_empty": 0.1,
                             "inner_shape": (6, 5), "display": False,
                             "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}]}, (6, 5), range(12)),
    ("padded_7x5_in_10x7", {"inner_shape": (7, 5), "prop_empty": 0.6, "prop_feats": 0.4,
                            "start_all_orders": [{"ingredients": ["onion", "onion", "onion"]}],
                            "display": False}, (10, 7), range(12)),
    ("padded_named", {"layout_name": "cramped_room"}, (8, 6), range(6)),
]


def gen_random_start_host(ns):
    """get_random_start_state_fn of the reference under np.random.seed(k): to_dict() of four consecutive draws."""
    out = {}
    for name in ("cramped_room", "counter_circuit"):
        m = refboot.make_mdp(ns, name)
        for pos, thr in ((True, 0.0), (False, 0.7), (True, 0.5)):
            for seed in range(4):
                refboot.use_mdp(ns, m)
                np.random.seed(seed)
                f = m.get_random_start_state_fn(random_start_pos=pos, rnd_obj_prob_thresh=thr)
                out["%s|%d|%s|%d" % (name, int(pos), thr, seed)] = [jsonable(f().to_dict()) for _ in range(4)]
    with open(os.path.join(GOLD, "random_start_host.json"), "w") as fh:
        json.dump(out, fh, sort_keys=True)
    print("random_start_host: %d seeded draws" % (4 * len(out)))


def gen_layoutgen(ns):
    """LayoutGenerator outputs of the reference under np.random.seed(k): terrain rows + start cells."""
    import copy
    import importlib

    lg = importlib.import_module("overcooked_ai_py.mdp.layout_generator")
    out = {}
    for name, params, outer, seeds in LAYOUTGEN_CASES:
        rows, starts = [], []
        for k in seeds:
            np.random.seed(k)
            gen = lg.LayoutGenerator(lg.MDPParamsGenerator.from_fixed_param(copy.deepcopy(params)), outer_shape=outer)
            m = gen.generate_padded_mdp()
            rows.append(["".join(r) for r in m.terrain_mtx])
            starts.append(list(m.start_player_positions))
        out[name + "__terrain"] = np.array(rows)
        out[name + "__starts"] = np.array(starts, dtype=np.int16)
        out[name + "__case"] = np.array(json.dumps({"params": params, "outer_shape": list(outer), "seeds": list(seeds)}))
        print("layoutgen %s: %d layouts, e.g. %s" % (name, len(rows), rows[0]))
    np.savez_compressed(os.path.join(GOLD, "layout_generator.npz"), **out)


def main():
    os.makedirs(GOLD, exist_ok=True)
    ns = refboot.boot()
    t0 = time.time()
    only = sys.argv[1:]
    if not only or "dynamics" in only:
        gen_dynamics_mdp_test(ns)
    if not only or "traces" in only:
        for i, (name, layout, params, eps, steps) in enumerate(TRACE_LAYOUTS):
            gen_traces(ns, name, layout, params, eps, steps, seed=1000 + i)
    if not only or "greedy" in only:
        gen_greedy_cramped_room(ns)
    if not only or "luts" in only:
        gen_planner_luts(ns)
    if not only or "human" in only:
        gen_human_2020(ns)
    if not only or "potential" in only:
        gen_potential(ns)
    if not only or "config1" in only:
        gen_config1(ns)
    if not only or "randstart" in only:
        gen_random_start_host(ns)
    if not only or "layoutgen" in only:
        gen_layoutgen(ns)
    print("done in %.1fs" % (time.time() - t0))


if __name__ == "__main__":
    main()
