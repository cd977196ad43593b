"""The rollout driver's configuration table (tests/test_gpu_rollout_forms.py) covers every axis value, every pair of values of
two axes (unless the pair is refused by the constructor, with the test that shows it, or cannot occur), every
constructor argument of SelfPlayRollout and AgentPairRollout and every argument of their collect(); and the refusals it
names exist."""
import inspect
import itertools
from types import SimpleNamespace

import pytest
import torch

import test_gpu_rollout_forms as G
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SelfPlayRollout
from test_policy_forms_cpu import defined_tests

SHARED = [a for a in G.AXES if not any(a in axes for axes in G.CLASS_AXES.values())]


def _matches(rule, case):
    a, va, b, vb = rule[:4]
    ok = lambda v, x: v == "*" or x == v or (isinstance(v, tuple) and x in v)
    return a in case and b in case and ok(va, case[a]) and ok(vb, case[b])


def _axes(case):
    return {k: v for k, v in case.items() if k in G.AXES}


def _excused(a, va, b, vb):
    probe = {a: va, b: vb}
    return any(_matches(r, probe) for r in G.REFUSED + G.NOT_APPLICABLE)


def test_every_case_is_well_formed():
    for name, case in G.CONFIGURATIONS.items():
        c = _axes(case)
        own = G.CLASS_AXES[c["class"]]
        want = set(SHARED) | set(own)
        if c.get("partner") == "none":
            want.discard("bc_factor")
        assert set(c) == want, (name, sorted(set(c) ^ want))
        for k, v in c.items():
            assert v in G.AXES[k], (name, k, v)
        for rule in G.REFUSED + G.NOT_APPLICABLE:
            assert not _matches(rule, c), (name, rule)
        n = case["n"]
        assert 97 <= n <= 301 and n % 32 and 17 <= case["T"] <= 30 and 7 <= case["horizon"] <= 13, name


def test_every_value_of_every_axis_has_a_case():
    seen = {k: set() for k in G.AXES}
    for case in G.CONFIGURATIONS.values():
        for k, v in _axes(case).items():
            seen[k].add(v)
    missing = {k: sorted(set(v) - seen[k]) for k, v in G.AXES.items() if set(v) - seen[k]}
    assert not missing, "axis values without a case: %s" % missing


def test_every_pair_of_values_has_a_case_or_a_reason():
    covered = set()
    for case in G.CONFIGURATIONS.values():
        c = _axes(case)
        for a, b in itertools.combinations(sorted(c), 2):
            covered.add((a, c[a], b, c[b]))
    missing = []
    for a, b in itertools.combinations(sorted(G.AXES), 2):
        for va in G.AXES[a]:
            for vb in G.AXES[b]:
                if (a, va, b, vb) not in covered and not _excused(a, va, b, vb):
                    missing.append("%s=%s with %s=%s" % (a, va, b, vb))
    assert not missing, "pairs of axis values with no case, no refusal and no reason: %s" % missing


def test_every_constructor_argument_belongs_to_an_axis_and_some_case_passes_it():
    """A new argument fails here until it is given an axis (or, for the few no axis varies, listed with its reason) and a
    case passes it."""
    params = set()
    for cls in (SelfPlayRollout, AgentPairRollout):
        params |= set(inspect.signature(cls.__init__).parameters) - {"self"}
    listed = set(G.PARAMETERS) | set(G.NOT_AN_AXIS)
    assert not set(G.PARAMETERS) & set(G.NOT_AN_AXIS)
    assert params == listed, ("constructor arguments not listed: %s; listed but gone: %s"
                              % (sorted(params - listed), sorted(listed - params)))
    assert set(G.NOT_AN_AXIS) == {"use_graph", "seed", "reward_shaping_factor", "max_seq_len"}
    for p, axis in G.PARAMETERS.items():
        assert axis in G.AXES, (p, axis)
    passed = set().union(*(G.passed_arguments(c) for c in G.CONFIGURATIONS.values()))
    assert params <= passed, "constructor arguments no case passes: %s" % sorted(params - passed)


def test_every_collect_argument_belongs_to_an_axis_or_has_a_reason():
    """A new collect() argument fails here until it is given an axis (or listed with the reason no axis varies it); the
    flag of the horizon bootstrap is passed by some case that collects."""
    params = set()
    for cls in (SelfPlayRollout, AgentPairRollout):
        params |= set(inspect.signature(cls.collect).parameters) - {"self"}
    assert not set(G.COLLECT_PARAMETERS) & set(G.COLLECT_NOT_AN_AXIS)
    listed = set(G.COLLECT_PARAMETERS) | set(G.COLLECT_NOT_AN_AXIS)
    assert params == listed, ("collect() arguments not listed: %s; listed but gone: %s"
                              % (sorted(params - listed), sorted(listed - params)))
    for p, axis in G.COLLECT_PARAMETERS.items():
        assert axis in G.AXES, (p, axis)
    assert any(c["bootstrap_horizon"] == "on" and c.get("agent0") not in G.SCRIPTED for c in G.CONFIGURATIONS.values())


def test_greedy_cases_play_qualifying_layouts():
    """GreedyHumanModel plays layouts of one 3-onion order only; the 9x5 grid has one such layout, so no pool there."""
    from overcooked_ai_b200 import greedy, layout

    for name, case in G.CONFIGURATIONS.items():
        if not G.is_greedy(case):
            continue
        single, pool = G.GREEDY_GRIDS[case["path"]]
        assert case["starts"] in (("fixed", "random") if pool is None else ("pool", "pool_redraw") if single is None else
                                  ("fixed", "random", "pool", "pool_redraw")), name
        for l in ([single] if single else []) + (pool or []):
            greedy.check_layout(layout.compile_layout(l))


def test_staggered_timesteps_end_some_warps_partly():
    for n, horizon in ((97, 7), (127, 13), (113, 10)):
        t = G.staggered_timesteps(n, horizon)
        assert ((0 <= t) & (t < horizon)).all() and (t == 0).sum() > 0.9 * n
        warps = [t[k:k + 32] for k in range(0, n, 32)]
        assert (warps[0] == 0).all() and all((w != 0).sum() == 1 for w in warps[1:]) and (t == horizon - 1).any()


def test_every_refusal_names_a_test_that_exists():
    for rule in G.REFUSED:
        module, test = rule[4].split("::")
        assert test in defined_tests(module), "%s names %s, which does not exist" % (rule[:4], rule[4])
    for rule in G.REFUSED + G.NOT_APPLICABLE:
        for axis, value in ((rule[0], rule[1]), (rule[2], rule[3])):
            values = value if isinstance(value, tuple) else () if value == "*" else (value,)
            assert axis in G.AXES and set(values) <= set(G.AXES[axis]), rule


def _env(n=4):
    return SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=n)


def test_selfplay_refuses_a_float32_lstm_learner():
    with pytest.raises(AssertionError, match="K11"):
        SelfPlayRollout(_env(), model=RllibLSTMShapedCNN(5, 4), autocast_dtype=None)


def test_selfplay_refuses_population_play_on_a_9x5_grid():
    """A 9x5 grid's first layer (9 x 5 x 25 = 1125 outputs, padded to 1136) is not a multiple of 64: no K7, so no
    population play, on the grid the K2 -> library -> draw cases run on."""
    env = SimpleNamespace(layouts=[SimpleNamespace(width=9, height=5)], device=torch.device("cpu"), n_layouts=1, n_envs=8)
    two = [RllibShapedCNN(9, 5), RllibShapedCNN(9, 5)]
    with pytest.raises(AssertionError, match="needs K7.*1 layouts on a 9x5 grid"):
        SelfPlayRollout(env, two, pair_weights=[[1.0, 1.0], [1.0, 1.0]])
    with pytest.raises(AssertionError, match="needs K7.*1 layouts on a 9x5 grid"):
        SelfPlayRollout(env, two, pairs=torch.zeros((8, 2), dtype=torch.int32))


def test_agent_pair_refuses_a_float32_lstm_agent_1():
    with pytest.raises(AssertionError, match="K11"):
        AgentPairRollout(_env(), (RllibShapedCNN(5, 4), RllibLSTMShapedCNN(5, 4)), autocast_dtype=None)
    with pytest.raises(AssertionError, match="K11"):
        AgentPairRollout(_env(), (BCPolicy(), RllibLSTMShapedCNN(5, 4)), autocast_dtype=None)
