"""collect(bootstrap_horizon=True) on the device: ovc_gae_horizon and its one-view form against a float32 loop of their
recurrence, ovc_horizon_rows against numpy, and whole windows of every learner configuration against the same collect()
without the flag, the recurrence on the batch's own tensors and the learner's value of the oracle's terminal states."""
import numpy as np
import pytest
import torch

from oracle import cpu
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.greedy import GreedyHumanModel
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibShapedCNN, SelfPlayRollout, records_forward
from ppo_reference import gae_horizon_f32
from test_gpu_bc_partner import POOL_5X4

pytestmark = pytest.mark.gpu

GAMMA, LAM = 0.99, 0.95

# the device entry points of csrc/libovc_horizon.so -> the tests that launch them (tests/test_horizon_bootstrap_cpu.py
# checks the table against the compiled library)
KERNELS = {
    "ovc::horizon_rows_kernel": ("test_horizon_rows_against_numpy", "test_collect_with_the_horizon_bootstrap"),
    "ovc::gae_horizon_kernel<float2>": ("test_gae_horizon_equals_the_float32_loop",),
    "ovc::gae_horizon_kernel<float>": ("test_gae_horizon_equals_the_float32_loop",),
}


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _done_patterns(T, n, rng):
    """dones [T, n] with, per environment: episode ends at t = 0, at T - 1, on consecutive steps, never, and random."""
    d = (rng.rand(T, n) < 0.15).astype(np.uint8)
    d[:, 0::5] = 0  # never
    d[0, 1::5] = 1
    d[T - 1, 2::5] = 1
    if T > 1:
        d[T // 2:T // 2 + 2, 3::5] = 1
    return d


# ------------------------------------------------------------------------------------------------ the GAE kernels


@pytest.mark.parametrize("T", [1, 2, 7, 16, 17, 60])
def test_gae_horizon_equals_the_float32_loop(T):
    """Both forms at an odd environment count, against the loop bit for bit; with every terminal value 0, against ovc_gae /
    ovc_gae_view bit for bit."""
    n = 301
    rng = np.random.RandomState(T)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    d = _done_patterns(T, n, rng)
    for one_view in (False, True):
        R = n if one_view else 2 * n
        r = rng.uniform(-2, 5, size=(T, R)).astype(np.float32)
        v = rng.uniform(-3, 3, size=(T, R)).astype(np.float32)
        tv = rng.uniform(-3, 3, size=(T, R)).astype(np.float32)
        last = rng.uniform(-3, 3, size=R).astype(np.float32)
        for terminal in (tv, np.zeros_like(tv)):
            adv = torch.full((T, R), float("nan"), device="cuda")
            tgt = torch.full((T, R), float("nan"), device="cuda")
            env.gae_horizon(_dev(r, torch.float32), _dev(v, torch.float32), _dev(d, torch.uint8), _dev(terminal, torch.float32),
                            _dev(last, torch.float32), GAMMA, LAM, adv, tgt, one_view=one_view)
            want_a, want_t = gae_horizon_f32(r, v, d, terminal, last, GAMMA, LAM)
            assert np.array_equal(_np(adv).view(np.int32), want_a.view(np.int32)), (one_view, T)
            assert np.array_equal(_np(tgt).view(np.int32), want_t.view(np.int32)), (one_view, T)
        # terminal values 0: the kernel without the bootstrap
        args = (_dev(r, torch.float32), _dev(v, torch.float32), _dev(d, torch.uint8), _dev(last, torch.float32), GAMMA, LAM)
        if one_view:
            a0, t0 = torch.empty((T, R), device="cuda"), torch.empty((T, R), device="cuda")
            env.gae_view(*args, a0, t0)
        else:
            a0, t0 = env.gae(*args)
        assert torch.equal(a0.view(-1).view(torch.int32), adv.view(-1).view(torch.int32)) and torch.equal(t0, tgt), (one_view, T)
    # the window holds every pattern
    assert d[0, 1::5].all() and d[T - 1, 2::5].all() and not d[:, 0::5].any()


# ------------------------------------------------------------------------------------------------ the compaction


@pytest.mark.parametrize("done", ["none", "all", "some"])
@pytest.mark.parametrize("mode", ["selfplay", "mixed_seats", "one_view"])
def test_horizon_rows_against_numpy(mode, done):
    n = 333
    rng = np.random.RandomState(len(mode) + len(done))
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400, rnd_obj_prob_thresh=0.5, random_start_pos=True, seed=3)
    for _ in range(3):
        env.step(_dev(rng.randint(0, 6, size=(n, 2)), torch.int32))
    d = {"none": np.zeros(n), "all": np.ones(n), "some": rng.rand(n) < 0.3}[done].astype(np.int32) * rng.randint(1, 3, n)
    env.done.copy_(_dev(d, torch.int32))
    seats = None if mode == "selfplay" else rng.randint(-1 if mode == "mixed_seats" else 0, 2, n).astype(np.int32)
    one_view = mode == "one_view"
    R = n if one_view else 2 * n
    recs, view, jrow = (torch.full(s, -7, dtype=torch.int32, device="cuda") for s in ((R, env.state_words), (R,), (R,)))
    rng_out = torch.full((2,), -7, dtype=torch.int32, device="cuda")
    values = torch.full((R,), float("nan"), device="cuda")
    env.horizon_rows(None if seats is None else _dev(seats, torch.int32), one_view, recs, view, jrow, rng_out, values)
    want = []  # (output row, view, environment)
    for e in np.nonzero(d)[0]:
        ps = -1 if seats is None else seats[e]
        views = [1 - ps] if one_view or ps >= 0 else [0, 1]
        want += [(e if one_view else 2 * e + v, v, e) for v in views]
    count = int(rng_out[1])
    assert int(rng_out[0]) == 0 and count == len(want)
    assert (_np(values) == 0).all()
    state = _np(env.state)
    got_j, got_v, got_r = _np(jrow)[:count], _np(view)[:count], _np(recs)[:count]
    order = np.argsort(got_j)
    assert np.array_equal(got_j[order], [w[0] for w in want]) and np.array_equal(got_v[order], [w[1] for w in want])
    assert np.array_equal(got_r[order], state[[w[2] for w in want]].reshape(-1, env.state_words))
    assert (_np(jrow)[count:] == -7).all()


# ------------------------------------------------------------------------------------------------ whole windows


def _env(layouts="cramped_room", **kw):
    return lambda: BatchedOvercookedEnv(layouts, 77, horizon=5, auto_reset=True, **kw)


RANDOM = dict(random_start_pos=True, rnd_obj_prob_thresh=0.4, seed=11)
POOL = dict(random_layout=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=5)
LIBRARY = dict(fused_first_layer=False, fused_wide=False, fused_tail=False)

# name -> (environment, class, keyword arguments of the rollout given the models (learner A, frozen B, BC, greedy))
CASES = {
    "selfplay": (_env(), "sp", lambda m: dict()),
    "selfplay_phi_random_starts": (_env(**RANDOM), "sp", lambda m: dict(use_phi=True)),
    "selfplay_library": (_env(), "sp", lambda m: dict(LIBRARY)),
    "selfplay_pool": (_env(POOL_5X4, **POOL), "sp", lambda m: dict()),
    "bc_partner": (_env(**RANDOM), "sp", lambda m: dict(partner=m["bc"], bc_factor=1.0)),
    "greedy_partner_phi": (_env(), "sp", lambda m: dict(partner=m["greedy"], bc_factor=0.5, use_phi=True)),
    "frozen_partner": (_env(), "sp", lambda m: dict(partner=m["B"], bc_factor=1.0)),
    "mixture": (_env(**RANDOM), "sp", lambda m: dict(partner=m["B"], bc_factor=0.5)),
    "mixture_library": (_env(), "sp", lambda m: dict(partner=m["B"], bc_factor=0.5, **LIBRARY)),
    "population": (_env(), "sp", lambda m: dict(partner=[m["B"], m["bc"]], bc_factor=0.5)),
    "pair_random_seats": (_env(**RANDOM), "pair", lambda m: dict(agents=(m["A"], m["bc"]), random_seats=True)),
    "pair_greedy_phi": (_env(), "pair", lambda m: dict(agents=(m["A"], m["greedy"]), random_seats=True, use_phi=True)),
    "pair_fixed_swap": (_env(), "pair", lambda m: dict(agents=(m["A"], m["B"]), swap=_dev(np.arange(77) % 2, torch.int32))),
    "pair_library_pool": (_env(POOL_5X4, **POOL), "pair", lambda m: dict(agents=(m["A"], m["B"]), random_seats=True)),
}


def _rollout(case, models, graph):
    make_env, kind, kw = CASES[case]
    env, kw = make_env(), kw(models)
    if kind == "sp":
        return SelfPlayRollout(env, model=models["A"], seed=7, use_graph=graph, **kw)
    agents = kw.pop("agents")
    return AgentPairRollout(env, agents, seed=7, use_graph=graph, **kw)


SAME = ("states", "actions", "logp", "values", "rewards", "dones", "last_values", "partner_seat", "partner_member", "pair")


def _snapshot(b):
    out = {k: getattr(b, k).clone() for k in SAME + ("advantages", "value_targets") if getattr(b, k) is not None}
    out["episodes"] = [t.clone() for t in b.episodes.tensors()]
    if b.terminal_values is not None:
        out["terminal_values"] = b.terminal_values.clone()
    return out


def _bits_equal(a, b):
    if isinstance(a, list):
        return len(a) == len(b) and all(_bits_equal(x, y) for x, y in zip(a, b))
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(-1).view(torch.uint8),
                                                                     b.contiguous().view(-1).view(torch.uint8))


def _live(r):
    return [r.env.state, r.ret_sparse] + r.stats.state_tensors() + r._live()


def _watch(r):
    """Record the terminal records, dones and joint actions of every value pass of ``r`` (eager only)."""
    seen = []
    inner = r._terminal_values

    def wrapped(out):
        joint = r.actions if isinstance(r, AgentPairRollout) else None
        seen.append((r.env.state.clone(), r.env.done.clone(), None if joint is None else joint.clone()))
        inner(out)
    r._terminal_values = wrapped
    return seen


def _check_terminal_values(r, b, seen, model):
    """terminal_values: 0 off the learner rows of the ended environments; there, the learner's value (records_forward) of
    the oracle's terminal state, rebuilt from states[t] and the joint action."""
    env, N = r.env, r.env.n_envs
    T = b.dones.shape[0]
    assert len(seen) == T
    tv, mask = _np(b.terminal_values), _np(b.learner_mask).astype(bool)
    dones = _np(b.dones).astype(bool)
    rows_per_env = 1 if b.one_view else 2
    ended = np.repeat(dones, rows_per_env, axis=1) & mask
    assert (tv[~ended] == 0).all()
    checked = 0
    for t in range(T):
        state, done, joint = seen[t]
        idx = np.nonzero(dones[t])[0]
        assert np.array_equal(_np(done) != 0, dones[t])
        if len(idx) == 0:
            continue
        acts = _np(b.actions[t]).reshape(N, 2) if joint is None else _np(joint)
        recs = np.ascontiguousarray(_np(b.states[t])[idx])
        cpu.step(env._tab_host, env._starts_host, recs, np.ascontiguousarray(acts[idx]), horizon=env.horizon, flags=0)
        assert np.array_equal(recs, _np(state)[idx]), t
        with torch.no_grad():
            d_recs = _dev(recs, torch.int32)
            if b.one_view:
                seat = _dev(_np(b.partner_seat[t])[idx], torch.int32)
                _, want = records_forward(model, env, d_recs, seat=1, swap=seat)
                got = tv[t][idx]
            else:
                _, want = records_forward(model, env, d_recs)
                got = tv[t].reshape(N, 2)[idx].reshape(-1)
                keep = mask[t].reshape(N, 2)[idx].reshape(-1)
                want, got = _np(want)[keep], got[keep]
        want = np.asarray(want.cpu() if torch.is_tensor(want) else want)
        assert np.abs(got - want).max() <= 0.03 * np.abs(want).max() + 1e-3, t
        checked += len(want)
    return checked


@pytest.mark.parametrize("case", sorted(CASES))
def test_collect_with_the_horizon_bootstrap(case):
    """Windows of 7 transitions at horizon 5, with a third of the environments reset one step out of phase: the eager and
    the graph collect(bootstrap_horizon=True) equal collect() without it in every other field, the environments, counters
    and statistics; their advantages are the recurrence on the batch's own tensors; their terminal values are the
    learner's value of the oracle's terminal states."""
    torch.manual_seed(len(case))
    models = dict(A=RllibShapedCNN(5, 4), B=RllibShapedCNN(5, 4), bc=BCPolicy(), greedy=GreedyHumanModel())
    runs = {k: _rollout(case, models, graph) for k, graph in (("plain", False), ("eager", False), ("graph", True))}
    stagger = (torch.arange(77, device="cuda") % 3 == 0).to(torch.int32)
    for r in runs.values():
        r.run(2)
        r.env.reset(stagger)
        r.reset_state()
    seen = _watch(runs["eager"])
    checked = 0
    for w in range(2):
        seen.clear()
        got = {k: _snapshot(r.collect(7, GAMMA, LAM, bootstrap_horizon=k != "plain")) for k, r in runs.items()}
        plain, eager, graph = got["plain"], got["eager"], got["graph"]
        assert plain.keys() | {"terminal_values"} == eager.keys() == graph.keys()
        for k in plain:
            if k not in ("advantages", "value_targets"):
                assert _bits_equal(plain[k], eager[k]), (w, k)
        for k in eager:
            assert _bits_equal(eager[k], graph[k]), (w, k)
        for x, y, z in zip(*(_live(r) for r in runs.values())):
            assert torch.equal(x, y) and torch.equal(x, z), w
        b = runs["eager"]._batches[(7, False, "bootstrap_horizon")]
        want_a, want_t = gae_horizon_f32(_np(b.rewards), _np(b.values), _np(b.dones), _np(b.terminal_values), _np(b.last_values),
                                         GAMMA, LAM)
        assert np.array_equal(_np(b.advantages).view(np.int32), want_a.view(np.int32)), w
        assert np.array_equal(_np(b.value_targets).view(np.int32), want_t.view(np.int32)), w
        dones = _np(b.dones)
        assert dones.any() and len({tuple(np.nonzero(dones[:, e])[0]) for e in range(77)}) > 1  # ends at different t
        checked += _check_terminal_values(runs["eager"], b, seen, models["A"])
        assert not torch.equal(b.advantages, runs["plain"]._batches[(7, False)].advantages)
    assert checked > 0
    r = runs["eager"]
    fused = (r.agents[0] if isinstance(r, AgentPairRollout) else r)
    fused = fused.fused_first_layer and fused.fused_wide and fused.fused_tail
    assert r._horizon.fused == fused
    assert fused == ("library" not in case and "pool" not in case), case
