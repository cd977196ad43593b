"""The CUDA kernels on the limit layouts of ``limit_layouts.py`` (16x16 grids, 4 pots, 124 object cells, 128 floor cells, cook
times up to 16382, the grids around K7's shared-memory limit) against the oracle, bit for bit.  The oracle's host tables for 3-4
pots are restated independently in ``test_layout_limits_cpu.py``."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import limit_layouts as LL
import policy_reference as P
from helpers import lut_bytes
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from test_layout_limits_cpu import restated_tables

pytestmark = pytest.mark.gpu

IOS = [_native.IO_TMA_TENSOR, _native.IO_TMA_BULK, _native.IO_DIRECT]
DYN = {"L16": (LL.l16, LL.l16_states), "L16_old": (LL.l16_old, LL.l16_old_states), "L3P": (LL.l3p, LL.l3p_states),
       "thin_16x3": (LL.thin_16x3, None), "thin_3x16": (LL.thin_3x16, None)}


def _np(t):
    return t.cpu().numpy()


def _actions(rng, T, n, p_interact=0.4):
    a = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32)
    a[rng.rand(T, n, 2) < p_interact] = 5
    return a


def _start(name, n, thresh, seed, io=_native.IO_DEFAULT, horizon=40):
    """An environment on one limit layout from device-drawn random starts, every hand-built state planted in a few of its
    environments; the oracle's mirror of the same starts."""
    make, states = DYN[name]
    lay = make()
    env = BatchedOvercookedEnv(lay, n, horizon=horizon, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=thresh,
                               seed=seed, io=io)
    rs = cpu.random_start(seed, thresh, True)
    ref = np.zeros((n, env.state_words), np.int32)
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs)
    assert np.array_equal(_np(env.state), ref), "K4 random starts"
    if states is not None:
        hand = np.stack([L.pack_state(lay, s, 0, env.state_words) for s in states(lay).values()])
        idx = np.arange(0, n, 5)[: 4 * len(hand)]
        ref[idx] = np.tile(hand, (4, 1))[: len(idx)]
        ref[idx, 0] = np.arange(len(idx)) % horizon  # some of them reach the horizon during the run
        env.state.copy_(torch.from_numpy(ref))
    return env, ref, rs


@pytest.mark.parametrize("thresh", [0.5, 1.0])
@pytest.mark.parametrize("name", list(DYN))
def test_k1_every_record_io_vs_oracle(name, thresh):
    """K1 through each of its three record-I/O strategies, transition by transition, interact-biased play with auto-reset:
    rewards, events, dones and the record after every transition."""
    n, T = 331, 45
    for io in IOS:
        env, ref, rs = _start(name, n, thresh, 17, io=io)
        acts = _actions(np.random.RandomState(3), T, n)
        d = torch.from_numpy(acts).cuda()
        for t in range(T):
            want = cpu.step(env._tab_host, env._starts_host, ref, acts[t], horizon=40, flags=1, n_threads=4, rs=rs)
            got = env.step(d[t])
            for g, w in zip(got, want):
                assert np.array_equal(_np(g), w), (io, t)
            assert np.array_equal(_np(env.state), ref), (io, t)


@pytest.mark.parametrize("thresh", [0.5, 1.0])
@pytest.mark.parametrize("name", list(DYN))
def test_k5_launch_lengths_vs_oracle(name, thresh):
    """K5 in launches of 2, 7 and 4096 transitions and in one launch (a 1-transition rollout runs K1): rewards, events, dones
    of every transition and the record after every launch."""
    n, T = 517, 90
    acts = _actions(np.random.RandomState(5), T, n)
    for chunk in (2, 7, 4096, 0):
        env, ref, rs = _start(name, n, thresh, 29)
        d = torch.from_numpy(acts).cuda()
        step = chunk if chunk else T
        for t0 in range(0, T, step):
            t1 = min(T, t0 + step)
            want = cpu.rollout(env._tab_host, env._starts_host, ref, acts[t0:t1], horizon=40, flags=1, n_threads=4, rs=rs)
            got = env.rollout(d[t0:t1].contiguous())
            for g, w in zip(got, want):
                assert np.array_equal(_np(g), w), (chunk, t0)
            assert np.array_equal(_np(env.state), ref), (chunk, t0)
    mask = (np.random.RandomState(1).rand(n) < 0.4).astype(np.int32)  # K4: a masked reset redraws exactly those
    env.reset(torch.from_numpy(mask).cuda())
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs, mask=mask)
    assert np.array_equal(_np(env.state), ref)


def test_long_cook_16382_inside_and_across_launches():
    """Every pot starts a 16382-step soup at tick 0; about 16 500 mostly-STAY transitions.  The soups are ready for the
    interacts of transition 16382.  One launch and launches of 4096 put that transition inside a launch (with the clock reloaded
    at three boundaries while the soups cook); launches of 8191 start a launch on it (the soup is loaded at tick == cook time);
    launches of 16381 end one transition before it (loaded at cook time - 1).  The first eight environments interact with
    dishes around it."""
    lay = LL.l16()
    n, T = 48, 16500
    pots = [LL.soup(p, LL.OT, 0) for p in lay.pot_locations]
    rec = L.pack_state(lay, LL._state(lay, [((1, 2), LL.W, "dish"), ((6, 1), LL.N, "dish")], pots))
    st0 = np.repeat(rec[None], n, 0)
    rng = np.random.RandomState(9)
    acts = np.full((T, n, 2), 4, np.int32)
    move = rng.rand(T, n, 2) < 0.01
    acts[move] = rng.randint(0, 6, size=int(move.sum()))
    acts[:, :8] = 4  # the first eight environments stand still, then interact around the ready tick with their dishes
    acts[16370:16400, :8] = 5
    ref = st0.copy()
    tab, starts, _ = L.build_tables([lay])
    want = cpu.rollout(tab, starts, ref, acts, horizon=0, n_threads=4)
    assert (want[1] == 11).any(), "a soup was picked up once ready"
    for chunk in (T, 4096, 8191, 16381):
        env = BatchedOvercookedEnv(lay, n, horizon=0)
        env.state.copy_(torch.from_numpy(st0))
        d = torch.from_numpy(acts).cuda()
        for t0 in range(0, T, chunk):
            t1 = min(T, t0 + chunk)
            got = env.rollout(d[t0:t1].contiguous())
            for g, w in zip(got, want):
                assert np.array_equal(_np(g), w[t0:t1]), (chunk, t0)
        assert np.array_equal(_np(env.state), ref), chunk
    ticks = [(int(ref[e, 4 + k]) >> 8) & 0x3FFF for e in range(8, n) for k in range(4)]
    assert L.MAX_TICK + 1 in ticks  # ready soups stop at tick == cook time


def _mixed_states(name, n=400, thresh=0.5, T=60):
    env, ref, rs = _start(name, n, thresh, 41, horizon=400)
    acts = _actions(np.random.RandomState(7), T, n)
    env.rollout(torch.from_numpy(acts).cuda())
    return env, _np(env.state).copy()


def _swap_views(a, swap):
    a = a.copy()
    a[swap] = a[swap][:, ::-1]
    return a


@pytest.mark.parametrize("name", ["L16", "L3P", "thin_16x3", "thin_3x16"])
def test_k2_lossless_encoding_every_dtype(name):
    """K2 against cpu.encode_lossless with view_swap: float32 / int32 equal; bfloat16 equal to the round-to-nearest-even
    bfloat16 of the oracle's values (cook times above 256); uint8 refused where a cook time exceeds 255.  On a 16x16 fp32 grid
    one observation is 53 KB (one environment per tile)."""
    env, st = _mixed_states(name)
    lay = env.layouts[0]
    want = cpu.encode_lossless(env._tab_host, st, lay.width, lay.height, 400)
    swap = (np.random.RandomState(2).rand(env.n_envs) < 0.5)
    vs = torch.from_numpy(swap.astype(np.int32)).cuda()
    want_s = _swap_views(want, swap)
    assert np.array_equal(_np(env.lossless_state_encoding(dtype=torch.float32, view_swap=vs)), want_s.astype(np.float32))
    assert np.array_equal(_np(env.lossless_state_encoding(dtype=torch.int32, view_swap=vs)), want_s)
    bf = _np(env.lossless_state_encoding(dtype=torch.bfloat16, view_swap=vs).float())
    assert np.array_equal(bf, P.bf16(want_s))
    if name == "L16":
        assert (want > 256).any() and not np.array_equal(P.bf16(want), want), "premise: values bf16 rounds"
    if lay.cook_time.max() > 255:
        with pytest.raises(ValueError, match="uint8"):
            env.lossless_state_encoding(dtype=torch.uint8)
    else:
        assert np.array_equal(_np(env.lossless_state_encoding(dtype=torch.uint8, view_swap=vs)).astype(np.int32), want_s)


def test_k2_uint8_of_over_cooked_soups_wraps_as_documented():
    """Cook times up to 255: uint8 is accepted; a hand-built over-cooked soup's negative cook time remaining is stored modulo
    256 (the documented case), everything else equals the oracle."""
    lay = LL.l16("L16_short", recipe_times=[1, 255, 200, 100, 30, 100])
    recs = np.stack([L.pack_state(lay, s) for s in LL.l16_states(lay).values()])
    env = BatchedOvercookedEnv(lay, len(recs), horizon=400)
    env.state.copy_(torch.from_numpy(recs))
    want = cpu.encode_lossless(env._tab_host, recs, 16, 16, 400)
    assert (want < 0).any() and want.max() > 127
    got = _np(env.lossless_state_encoding(dtype=torch.uint8))
    assert np.array_equal(got, (want & 0xFF).astype(np.uint8))
    assert np.array_equal(_np(env.lossless_state_encoding(dtype=torch.int32)), want)


@pytest.mark.parametrize("name", ["L16", "L16_old", "L3P", "thin_16x3", "thin_3x16"])
def test_k3_featurize_up_to_five_pots(name):
    """K3 with num_pots 0-5 against cpu.featurize; the pot blocks name the pots in the order of the independently restated
    planner table (bytes 2 and 3 of pot_order included)."""
    env, st = _mixed_states(name)
    lay = env.layouts[0]
    for num_pots in range(6):
        got = _np(env.featurize_state(num_pots=num_pots)).astype(np.float64)
        assert np.array_equal(got, cpu.featurize(env._tab_host, lut_bytes([lay]), st, num_pots)), num_pots
    flut, _ = restated_tables(lay)
    checked = 0
    for e in range(env.n_envs):
        for j in range(2):
            w = int(st[e, 1 + j]) & 0xFFFFFFFF
            x, y, o = w & 15, (w >> 4) & 15, (w >> 8) & 3
            for k in range(lay.n_pots):
                slot = int(flut["pot_order"][(y << 4) | x, o][k])
                if slot == L.NO_SLOT:
                    assert (got[e, j, 22 + 10 * k: 32 + 10 * k] == 0).all()
                    continue
                px, py = lay.slot_positions[slot]
                assert tuple(got[e, j, 30 + 10 * k: 32 + 10 * k]) == (px - x, py - y)
                checked += k >= 2
    assert checked > 0 or lay.n_pots <= 2


@pytest.mark.parametrize("gamma", [0.99, 0.9])
def test_k6_potential_partial_pots_and_16382_cook(gamma):
    """K6 against cpu.potential on every assignment of 0 / 1 / 2 ingredients to L16's four pots (all 81 partial_order rows),
    with a 16382-step soup cooking, and on random play."""
    lay = LL.l16()
    recs = []
    for code in range(81):
        cls = [(code // 3 ** k) % 3 for k in range(4)]
        objs = [LL.soup(p, {1: [LL.O1, LL.T1], 2: [LL.O2, LL.OT]}[c][(code + k) % 2], -1)
                for k, (p, c) in enumerate(zip(lay.pot_locations, cls)) if c]
        players = [((1, 2), LL.W, "onion" if code % 2 else None), ((6, 1), LL.N, "dish" if code % 5 else None)]
        recs.append(L.pack_state(lay, LL._state(lay, players, objs)))
        cooking = [LL.soup(lay.pot_locations[code % 4], LL.OT, code % 7)] + [o for o in objs if o.position != lay.pot_locations[code % 4]]
        recs.append(L.pack_state(lay, LL._state(lay, players, cooking)))
    recs += [L.pack_state(lay, s) for s in LL.l16_states(lay).values()]
    env = BatchedOvercookedEnv(lay, len(recs), horizon=400)
    env.state.copy_(torch.from_numpy(np.stack(recs)))
    pt, cl, gpow = L.build_potential_tables([lay], gamma)
    want = cpu.potential(env._tab_host, pt, cl, gpow, np.stack(recs))
    got = _np(env.potential(gamma))
    assert np.array_equal(got, want) and len(np.unique(want)) > 40
    for name in ("L16", "L3P"):
        env, st = _mixed_states(name)
        pt, cl, gpow = L.build_potential_tables(env.layouts, gamma)
        assert np.array_equal(_np(env.potential(gamma)), cpu.potential(env._tab_host, pt, cl, gpow, st))


# ------------------------------------------------------------------------------------------------------------------------- K7
def _max_smem():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def _k7_smem(cells, n_layouts, cpl=2):
    """encode_linear_smem (csrc/ovc_encfc.cuh) of the narrowest column slice, restated.  The kernel's own boundary is tested
    below (13x7 / 7x13 with 8 layouts accepted, 12x8 refused), so a drift of the formula from the kernel shows there."""
    cs = 32 * cpl
    return cells * 19 * cs * 2 + (n_layouts + 1) * cs * 4 + n_layouts * (16 * 4 + 2 * 4 + 128 * 2 + 256) + 16


def test_k7_shape_boundary_follows_its_shared_memory():
    cap = _max_smem()
    fits = [c for c in range(1, 257) if _k7_smem(c, 8) <= cap]
    assert 91 in fits and 96 not in fits  # 13x7 / 7x13 fit with 8 layouts; 12x8 / 16x6 do not with one
    assert _k7_smem(96, 1) > cap
    from overcooked_ai_b200.selfplay import fused_kernel_support

    # a network whose first layer is 128 wide: only the grid's table decides
    lin = lambda i, o: SimpleNamespace(in_features=i, out_features=o)
    net = SimpleNamespace(conv_as_linear=[lin(1, 128), lin(128, 64), lin(64, 64)], dense=[lin(64, 64)], n_actions=6)
    for (W, H), ok in (((13, 7), True), ((7, 13), True), ((12, 8), False), ((16, 6), False)):
        assert fused_kernel_support(net, W, H)[0] == ok, (W, H)
    # fused_kernel_support's shared-memory bound does not depend on the layout count; it agrees with the kernel's for 1 and
    # for 8 layouts on every grid shape up to 16x16 because no such grid has 92-95 cells
    for W in range(1, 17):
        for H in range(1, 17):
            fit1, fit8 = _k7_smem(W * H, 1) <= cap, _k7_smem(W * H, 8) <= cap
            assert fused_kernel_support(net, W, H)[0] == fused_kernel_support(net, W, H, 8)[0] == fit1 == fit8, (W, H)
    # the layout count has its own bound: ovc_encode_linear takes 1 and 8 layouts of a 5x4 grid and refuses 9
    pool = ["cramped_room", "cramped_room_tomato", "simple_o_t", "simple_tomato", "bonus_order_test", "mdp_test",
            "m_shaped_s", "simple_o", "cramped_room_o_3orders"]
    wt, bias = torch.zeros((520, 128), dtype=torch.bfloat16, device="cuda"), torch.zeros(128, device="cuda")
    for k in (1, 8, 9):
        env = BatchedOvercookedEnv(pool[:k], 2 * k + 1, horizon=40)
        try:
            env.encoded_linear(wt, bias)
            accepted = True
        except RuntimeError as e:
            assert "more than 8 layouts per call" in str(e)
            accepted = False
        assert fused_kernel_support(net, 5, 4, k)[0] == accepted == (k <= 8), k


def _k7_states(layouts, n):
    """Random play on 8 layouts of one shape, plus hand-built over-cooked soups (negative entries) and 16382-step soups."""
    env = BatchedOvercookedEnv(layouts, n, horizon=60, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=3)
    env.rollout(torch.from_numpy(_actions(np.random.RandomState(4), 50, n, 0.5)).cuda())
    st = _np(env.state).copy()
    lay = layouts[0]  # cook time 16382 for three onions, 3 for onion + tomato, 257 for a tomato
    W, H = lay.width, lay.height
    pa, pb = lay.pot_locations
    nxt = lambda p: (1, p[1]) if p[0] == 0 else (p[0] - 1, p[1])
    ori = lambda p: LL.W if p[0] == 0 else LL.E
    hand = [
        LL._state(lay, [(nxt(pa), ori(pa), None), (nxt(pb), ori(pb), (LL.O3, 16382))], [LL.soup(pa, LL.O3, 0), LL.soup(pb, LL.OT, 900)]),
        LL._state(lay, [(nxt(pa), ori(pa), "dish"), (nxt(pb), ori(pb), None)], [LL.soup(pa, LL.T1, 16382), LL.soup(pb, LL.O3, 16381)]),
    ]
    seg0 = np.flatnonzero(env.env_layout_host == 0)
    for i, s in enumerate(hand):
        st[seg0[i::len(hand)][:20]] = L.pack_state(lay, s, 0, env.state_words)
    env.state.copy_(torch.from_numpy(st))
    want = cpu.encode_lossless(env._tab_host, st, W, H, 60)
    assert want.min() < 0 and want.max() == L.MAX_TICK
    return env, st, want


@pytest.mark.parametrize("shape", [(13, 7), (7, 13)], ids=["13x7", "7x13"])
def test_k7_largest_grids_eight_layouts_bit_exact(shape):
    """K7 on the largest grids whose table fits, 8 layouts per call (one with a 16382-step soup, over-cooked soups with negative
    entries), view swap: equal to k7_reference bit for bit on certified dyadic operands."""
    W, H = shape
    env, st, obs = _k7_states(LL.k7_layouts(W, H), 8 * 97 + 5)
    rng = np.random.RandomState(W * 100 + H)
    n_in, n_out = W * H * 26, 128
    wt, bias = P.k7_operands(rng, n_in, n_out)
    rows20 = np.arange(n_in) % 26 == 20  # cook time remaining reaches 16382: small weights keep every sum exact
    wt[rows20] = P.dyadic(rng, (int(rows20.sum()), n_out), 7, [6], density=0.3)
    swap = np.random.RandomState(6).rand(env.n_envs) < 0.5
    rows = _swap_views(obs, swap).reshape(2 * env.n_envs, -1)
    for slope in (0.0, 0.25):
        want, certs = P.k7_reference(rows, wt, bias, slope)
        assert all(c.holds() for c in certs), "premise: certified exact accumulations"
        got = env.encoded_linear(torch.from_numpy(wt).float().cuda().to(torch.bfloat16), torch.from_numpy(bias).float().cuda(),
                                 neg_slope=slope, view_swap=torch.from_numpy(swap.astype(np.int32)).cuda())
        assert np.array_equal(_np(got.float()).astype(np.float64), want), slope


def test_k7_refuses_the_smallest_grid_beyond_and_collect_uses_the_library_path():
    """12x8 (96 cells): ovc_encode_linear returns OVC_E_UNSUPPORTED with a message, SelfPlayRollout runs K2 + library layers,
    and its logits and values equal the float64 CNN on the batch's observations."""
    from overcooked_ai_b200.selfplay import SelfPlayRollout

    lay = LL.k7_layouts(12, 8, 2)[1]
    n, T = 64, 6
    env = BatchedOvercookedEnv(lay, n, horizon=9, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.8, seed=3)
    wt = torch.zeros((12 * 8 * 26, 64), dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, dtype=torch.float32, device="cuda")
    out = torch.zeros((2 * n, 64), dtype=torch.bfloat16, device="cuda")
    lib = _native.lib()
    rc = lib.ovc_encode_linear(env.tables.data_ptr(), 1, env.state.data_ptr(), 0, wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n,
                               env.state_words, 12, 8, 400, 64, 0.2, 0)
    assert rc == -3 and b"does not fit shared memory" in lib.ovc_last_error()
    bound = int(lay.cook_time.max())
    model = P.exact_cnn(12, 8, seed=6, cook_time=bound).cuda()
    sp = SelfPlayRollout(env, model=model, use_graph=False, seed=2)
    assert not sp.fused_first_layer
    b = sp.collect(T, 0.99, 0.95, keep_logits=True)
    obs = _np(b.observations(torch.arange(T * n, device="cuda")))
    assert (obs <= P.plane_bounds(bound)).all()
    logits, values = P.cnn_forward64(model, obs)
    assert np.array_equal(_np(b.logits)[..., :6], logits.reshape(T, 2 * n, 6))
    assert np.array_equal(_np(b.values), values.reshape(T, 2 * n))
    assert len(np.unique(logits)) > 8
