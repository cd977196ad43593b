"""The greedy partner on the device (include/ovc_greedy.h): the kernel teacher-forced on the reference's GreedyHumanModel
games, bit for bit against the host restatement (tests/greedy_reference.py) on random reachable states of every qualifying
layout, and inside AgentPairRollout and SelfPlayRollout, whose environments must follow the CPU oracle on the drawn
actions."""
import copy

import numpy as np
import pytest
import torch

import greedy_reference as R
from helpers import GOLD
from oracle import cpu as oracle_cpu
from overcooked_ai_b200 import greedy as G
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN, SelfPlayRollout
from test_gpu_pair_collect import GAMMA, LAM, _check_window

pytestmark = pytest.mark.gpu

# every device entry point of libovc_greedy.so and the tests here that compare it with the restatement
KERNELS = {
    "ovc::greedy_actions_kernel": ("test_teacher_forced_on_the_reference_games", "test_random_states_of_every_layout_match_the_restatement",
                                   "test_agent_pair_follows_the_oracle_and_the_restatement"),
}


def _i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def test_teacher_forced_on_the_reference_games():
    """Step the environments with the golden's actions; both players' kernel actions equal the golden's at every step
    where the players moved or turned, and the restatement's (stuck draws included) at every step."""
    d = np.load(GOLD + "/greedy_cramped_room.npz")
    states, actions = d["states"], d["actions"]
    E, T = states.shape[:2]
    cl = L.compile_layout("cramped_room")
    env = BatchedOvercookedEnv("cramped_room", E, horizon=400, auto_reset=False)
    env.state.copy_(_i32(states[:, 0]))
    seed = 11
    players = [_i32(np.full(E, p)) for p in range(2)]
    prev = [torch.zeros(E, dtype=torch.int32, device="cuda") for _ in range(2)]
    counter = [torch.zeros(2, dtype=torch.int64, device="cuda") for _ in range(2)]
    refs = [R.GreedyReference([cl], seed, E) for _ in range(2)]
    out = torch.full((E, 2), -7, dtype=torch.int32, device="cuda")
    matched = stuck = 0
    for t in range(T):
        assert np.array_equal(env.state.cpu().numpy(), states[:, t]), t
        for p in range(2):
            env.greedy_actions(players[p], prev[p], counter[p], seed=seed ^ G.GREEDY_DRAW_SALT, out=out)
            got = out[:, p].cpu().numpy()
            assert np.array_equal(got, refs[p].act(states[:, t], np.full(E, p))), (t, p)
            assert prev[p].cpu().tolist() == refs[p].prev and int(counter[p][0]) == t + 1 and int(counter[p][1]) == 0
            for e in range(E):
                if t > 0 and R.players_key(states[e, t - 1]) == R.players_key(states[e, t]):
                    stuck += 1
                else:
                    assert got[e] == actions[e, t, p], (e, t, p)
                    matched += 1
        if t + 1 < T:
            env.step(_i32(actions[:, t]))
    assert matched == 3024 and stuck == 2 * 488


def _qualifying(old_dynamics):
    out = []
    for name in L.layout_names():
        try:
            cl = L.compile_layout(name, old_dynamics=old_dynamics)
            G.check_layout(cl)
        except (ValueError, AssertionError):
            continue
        out.append(cl)
    return out


def _pot_classes(layouts, recs):
    seen = set()
    for rec in recs:
        cl = layouts[int(rec[3]) & 0xFF]
        seen |= set(R.pot_states(cl, rec))
    return seen


@pytest.mark.parametrize("old_dynamics", [False, True], ids=["new", "old_dynamics"])
def test_random_states_of_every_layout_match_the_restatement(old_dynamics):
    """Random starts (positions, held objects, pots in every state) stepped by interact-heavy random actions, so objects
    lie on counters; per call a random player (or none), random episode ends and forced stuck steps.  Actions, the
    previous-state keys and the draw counter equal the restatement's, untouched entries stay untouched."""
    layouts = _qualifying(old_dynamics)
    per = 24
    n = per * len(layouts)
    env = BatchedOvercookedEnv(layouts, n, horizon=25, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=3)
    seed = 123
    ref = R.GreedyReference(layouts, seed, n)
    prev = torch.zeros(n, dtype=torch.int32, device="cuda")
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    rng = np.random.RandomState(4)
    seen_pots, counter_objs, stuck = set(), 0, 0
    for t in range(40):
        recs = env.state.cpu().numpy()
        player = rng.randint(-1, 2, size=n)
        done = (rng.rand(n) < 0.1).astype(np.int32)
        keys = np.array([R.state_key(r) for r in recs], np.int64)
        p_host = prev.cpu().numpy().astype(np.int64)
        force = rng.rand(n) < 0.3
        p_host[force] = keys[force]
        prev.copy_(_i32(p_host))
        ref.prev, ref.step = p_host.tolist(), int(counter[0])
        want = ref.act(recs, player, done)
        out = torch.full((n, 2), -7, dtype=torch.int32, device="cuda")
        env.greedy_actions(_i32(player), prev, counter, seed=seed ^ G.GREEDY_DRAW_SALT, done=_i32(done), out=out)
        got = out.cpu().numpy()
        on = player >= 0
        assert np.array_equal(got[on, player[on]], want[on]), t
        assert (got[on, 1 - player[on]] == -7).all() and (got[~on] == -7).all()
        assert prev.cpu().tolist() == [int(v) for v in ref.prev] and int(counter[0]) == t + 1
        stuck += int((on & force & (done == 0)).sum())
        seen_pots |= _pot_classes(layouts, recs)
        for r in recs:
            cl = layouts[int(r[3]) & 0xFF]
            counter_objs += int(((r[4 + cl.n_pots:4 + cl.n_slots] & 7) != 0).sum())
        acts = rng.randint(0, 6, size=(n, 2))
        acts[rng.rand(n, 2) < 0.35] = 5
        env.step(_i32(acts))
    assert {"empty", "1_items", "2_items", "cooking", "ready"} <= seen_pots, seen_pots
    if not old_dynamics:
        assert "3_items" in seen_pots
    assert counter_objs > 100 and stuck > 1000


def _greedy_players(pair, k, seats):
    """The players agent k holds this transition: fixed seats, swap, or the drawn seats (agent 1) and their complement."""
    n = pair.env.n_envs
    if pair.random_seats:
        s = pair.partner_seat.cpu().numpy()
        return s if k == 1 else 1 - s
    swap = np.zeros(n, np.int64) if pair.swap is None else (pair.swap.cpu().numpy() != 0).astype(np.int64)
    return seats[k] ^ swap


CONFIGS = {
    "ppo_greedy": dict(agents=("ppo", "greedy")),
    "greedy_ppo_swap": dict(agents=("greedy", "ppo"), swap=True),
    "ppo_greedy_random_seats": dict(agents=("ppo", "greedy"), random_seats=True),
    "greedy_greedy": dict(agents=("greedy", "greedy"), swap=True),
}


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_agent_pair_follows_the_oracle_and_the_restatement(name, graph):
    """Whole run() transitions: every greedy action equals the restatement's on the state before it (its seats, the
    previous transition's episode ends, its own draw counter), and the environments follow the CPU oracle."""
    cfg = CONFIGS[name]
    n, horizon, T, seed = 203, 11, 30, 9
    torch.manual_seed(2)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    agents = tuple(G.GreedyHumanModel() if a == "greedy" else RllibShapedCNN(5, 4) for a in cfg["agents"])
    swap = _i32(np.random.RandomState(1).randint(0, 2, n)) if cfg.get("swap") else None
    pair = AgentPairRollout(env, agents, swap=swap, seed=seed, use_graph=graph, random_seats=cfg.get("random_seats", False))
    cl = env.layouts[0]
    refs = {k: R.GreedyReference([cl], seed, n) for k, a in enumerate(cfg["agents"]) if a == "greedy"}
    st = env.state.cpu().numpy().copy()
    done = env.done.cpu().numpy().copy() * 0  # no previous transition
    for t in range(T):
        players = {k: _greedy_players(pair, k, (0, 1)) for k in refs}
        pair.run(1)
        acts = pair.actions.cpu().numpy()
        for k, ref in refs.items():
            want = ref.act(st, players[k], done)
            assert np.array_equal(acts[np.arange(n), players[k]], want), (t, k)
        _, _, dn, _ = oracle_cpu.step(env._tab_host, env._starts_host, st, acts, horizon=horizon, flags=1)
        assert np.array_equal(env.state.cpu().numpy(), st), t
        done = dn.copy()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_agent_pair_collect_draws_what_run_draws(graph):
    """collect() next to a greedy partner with random seats plays the transitions run() plays: the same states, seats
    and learner actions."""
    n, T = 300, 25
    torch.manual_seed(6)
    A = RllibShapedCNN(5, 4)
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=10, auto_reset=True)
    p1 = AgentPairRollout(e1, (A, G.GreedyHumanModel()), seed=8, random_seats=True, use_graph=graph)
    p2 = AgentPairRollout(e2, (copy.deepcopy(A), G.GreedyHumanModel()), seed=8, random_seats=True, use_graph=graph)
    for w in range(2):
        b = p1.collect(T, GAMMA, LAM)
        rows = 2 * torch.arange(n, device="cuda") + (1 - b.partner_seat.long())
        for t in range(T):
            assert torch.equal(b.states[t], e2.state) and torch.equal(p2.partner_seat, b.partner_seat[t].int()), (w, t)
            p2.run(1)
            assert torch.equal(p2.actions.view(-1)[rows[t]], b.actions[t]), (w, t)
        assert torch.equal(e1.state, e2.state)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_selfplay_with_a_greedy_partner_at_bc_factor_0_is_selfplay(graph):
    n, T = 256, 20
    torch.manual_seed(3)
    A = RllibShapedCNN(5, 4)
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=9, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=9, auto_reset=True)
    sp1 = SelfPlayRollout(e1, model=A, seed=5, partner=G.GreedyHumanModel(), bc_factor=0.0, use_graph=graph)
    sp2 = SelfPlayRollout(e2, model=copy.deepcopy(A), seed=5, use_graph=graph)
    assert (sp1.partner_seat == -1).all()
    for w in range(2):
        b1, b2 = sp1.collect(T, GAMMA, LAM), sp2.collect(T, GAMMA, LAM)
        for k in ("states", "actions", "logp", "values", "rewards", "dones", "advantages", "value_targets"):
            assert torch.equal(getattr(b1, k), getattr(b2, k)), (w, k)
    sp1.run(7), sp2.run(7)
    assert torch.equal(sp1.actions, sp2.actions) and torch.equal(e1.state, e2.state)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_selfplay_with_a_greedy_partner_at_bc_factor_1_is_the_pair(graph):
    """PPO next to the greedy partner in SelfPlayRollout's drawn seats equals AgentPairRollout((learner, greedy),
    random_seats=True) on the learner's rows, the seats and the episode records."""
    n, horizon, T = 640, 12, 20
    torch.manual_seed(5)
    A = RllibShapedCNN(5, 4)
    e1 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    e2 = BatchedOvercookedEnv("cramped_room", n, horizon=horizon, auto_reset=True)
    sp = SelfPlayRollout(e1, model=copy.deepcopy(A), seed=4, partner=G.GreedyHumanModel(), bc_factor=1.0, use_graph=graph)
    pair = AgentPairRollout(e2, (A, G.GreedyHumanModel()), seed=4, random_seats=True, use_graph=graph)
    assert torch.equal(sp.partner_seat, pair.partner_seat)
    for w in range(2):
        bs, bp = sp.collect(T, GAMMA, LAM), pair.collect(T, GAMMA, LAM)
        _check_window(bs, bp, pair, False, with_seats=True)
        assert torch.equal(e1.state, e2.state), w
