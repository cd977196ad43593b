"""GPU parity tests: the CUDA kernels, called through the C ABI (ctypes, include/ovc_b200.h), against
the CPU oracle and the reference-generated golden fixtures.  Bit-exact everywhere (integer path;
the float32 outputs hold small integers)."""
import numpy as np
import pytest
import torch

from helpers import EVENT_MASK, GOLD, TRACE_FILES, TRACE_IDS, Trace, lut_bytes
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.batched import BatchedOvercookedEnv, EpisodeStats, HostRolloutPipeline

pytestmark = pytest.mark.gpu

IOS = [_native.IO_TMA_TENSOR, _native.IO_TMA_BULK, _native.IO_DIRECT]
IO_IDS = ["tma2d", "bulk1d", "direct"]
CLASSIC5 = ["cramped_room", "asymmetric_advantages", "coordination_ring", "forced_coordination", "counter_circuit"]


def _env_for_trace(tr, n, io, horizon=0, auto_reset=False):
    return BatchedOvercookedEnv(tr.layout, n, horizon=horizon, io=io, auto_reset=auto_reset)


def _np(t):
    return t.cpu().numpy()


@pytest.mark.parametrize("io", IOS, ids=IO_IDS)
@pytest.mark.parametrize("path", TRACE_FILES + [GOLD + "/dynamics_mdp_test.npz"], ids=TRACE_IDS + ["dynamics_mdp_test"])
def test_golden_transitions(path, io):
    """Every reference transition in the fixture, as one batch, through each record-I/O strategy."""
    tr = Trace(path)
    s0, a, s1, sparse, shaped, events = tr.flat()
    env = _env_for_trace(tr, len(s0), io)
    env.state.copy_(torch.from_numpy(s0))
    sp, sh, dn, ev = env.step(torch.from_numpy(a).cuda())
    assert np.array_equal(_np(env.state), s1)
    assert np.array_equal(_np(sp), sparse)
    assert np.array_equal(_np(sh), shaped)
    assert np.array_equal(_np(ev) & EVENT_MASK, events)
    assert not _np(dn).any()
    by_agent = _np(env.sparse_by_agent(ev))
    assert np.array_equal(by_agent.reshape(tr.sparse2.shape), tr.sparse2)


@pytest.mark.parametrize("chunk", [2, 7, 0], ids=["chunks_of_2", "chunks_of_7", "whole"])
@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_golden_trajectories_fused(path, chunk):
    """Every fixture trajectory through the fused rollout kernel K5, cut into launches of `chunk` transitions (0: one
    launch): rewards / events of every transition and the record after every launch.  Short launches put every
    cooking soup through the kernel's on-chip <-> record conversion at every possible tick."""
    tr = Trace(path)
    env = _env_for_trace(tr, tr.E, _native.IO_DEFAULT)
    env.state.copy_(torch.from_numpy(np.ascontiguousarray(tr.states[:, 0])))
    acts = torch.from_numpy(np.ascontiguousarray(tr.actions.transpose(1, 0, 2))).cuda()  # [T,E,2]
    step = chunk if chunk else tr.T
    for t0 in range(0, tr.T, step):
        t1 = min(tr.T, t0 + step)
        sp, sh, dn, ev = [_np(x) for x in env.rollout(acts[t0:t1].contiguous())]
        assert np.array_equal(_np(env.state), tr.states[:, t1]), "record after transitions %d..%d" % (t0, t1)
        assert np.array_equal(sp.T, tr.sparse[:, t0:t1])
        assert np.array_equal(sh.transpose(1, 0, 2), tr.shaped[:, t0:t1])
        assert np.array_equal(ev.transpose(1, 0, 2) & EVENT_MASK, tr.events[:, t0:t1])
        assert not dn.any()


def test_greedy_games_stepwise_and_fused():
    """5 GreedyHumanModel games on cramped_room (9 deliveries each): per-step launches, then the same
    games again through the fused T-step rollout kernel."""
    tr = Trace(GOLD + "/greedy_cramped_room.npz")
    acts = torch.from_numpy(np.ascontiguousarray(tr.actions.transpose(1, 0, 2))).cuda()  # [T,E,2]
    for mode in ("step", "rollout"):
        env = BatchedOvercookedEnv("cramped_room", tr.E, horizon=400)
        assert np.array_equal(_np(env.state), tr.states[:, 0])
        if mode == "step":
            sps, shs, evs = [], [], []
            for t in range(tr.T):
                sp, sh, dn, ev = env.step(acts[t])
                sps.append(_np(sp)), shs.append(_np(sh)), evs.append(_np(ev))
                if t + 1 < tr.T:
                    assert np.array_equal(_np(env.state), tr.states[:, t + 1])
            sp, sh, ev = np.stack(sps), np.stack(shs), np.stack(evs)
        else:
            sp, sh, dn, ev = [_np(x) for x in env.rollout(acts)]
            assert dn[-1].all() and not dn[:-1].any()
        assert np.array_equal(sp.T, tr.sparse) and sp.sum(0).tolist() == [180] * 5
        assert np.array_equal(sh.transpose(1, 0, 2), tr.shaped)
        assert np.array_equal(ev.transpose(1, 0, 2) & EVENT_MASK, tr.events)


def test_lossless_reference_golden_pickle():
    d = np.load(GOLD + "/greedy_cramped_room.npz")
    states = d["states"].reshape(-1, 16)
    env = BatchedOvercookedEnv("cramped_room", len(states), horizon=400)
    env.state.copy_(torch.from_numpy(states))
    want = d["lossless"].reshape(-1, 2, 5, 4, 26)
    for dt in (torch.float32, torch.uint8, torch.int32, torch.bfloat16):
        enc = env.lossless_state_encoding(dtype=dt)
        assert enc.dtype == dt and tuple(enc.shape) == (len(states), 2, 5, 4, 26)
        assert np.array_equal(_np(enc.float()).astype(np.int32), want.astype(np.int32))


@pytest.mark.parametrize("num_pots", [0, 1, 2])
def test_featurize_reference_golden_pickles(num_pots):
    d = np.load(GOLD + "/greedy_cramped_room.npz")
    states = d["states"].reshape(-1, 16)
    env = BatchedOvercookedEnv("cramped_room", len(states), horizon=400)
    env.state.copy_(torch.from_numpy(states))
    f = _np(env.featurize_state(num_pots=num_pots))
    exp = d["feat_%d" % num_pots].reshape(len(states), 2, -1)
    assert f.dtype == np.float32 and np.array_equal(f, exp.astype(np.float32))


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_golden_observations(path):
    tr = Trace(path)
    d = tr.data
    st = d["obs_states"]
    env = _env_for_trace(tr, len(st), 0, horizon=400)
    env.state.copy_(torch.from_numpy(st))
    enc = env.lossless_state_encoding(dtype=torch.float32)
    assert np.array_equal(_np(enc), d["obs_lossless"].astype(np.float32))
    enc8 = env.lossless_state_encoding(dtype=torch.uint8)
    assert np.array_equal(_np(enc8).astype(np.int16), d["obs_lossless"])
    for num_pots in (0, 1, 2, 3):
        f = _np(env.featurize_state(num_pots=num_pots))
        assert np.array_equal(f, d["obs_feat_%d" % num_pots].astype(np.float32)), num_pots


def _random_actions(rng, T, n, p_interact=0.3):
    a = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32)
    a[rng.rand(T, n, 2) < p_interact] = 5
    return a


@pytest.mark.parametrize("io", IOS, ids=IO_IDS)
@pytest.mark.parametrize("auto_reset", [False, True], ids=["noreset", "autoreset"])
def test_mixed_layout_rollout_vs_oracle(io, auto_reset):
    """5 classic layouts in one batch (BASELINE config 3 shape, small), ragged env count so the last
    tile is partial, horizon crossed: per-step kernel for the first part, fused rollout for the rest."""
    n, T, horizon = 5 * 811 + 3, 90, 60
    env = BatchedOvercookedEnv(CLASSIC5, n, horizon=horizon, io=io, auto_reset=auto_reset)
    assert env.state_words == 32
    rng = np.random.RandomState(7)
    acts = _random_actions(rng, T, n)
    ref_state = _np(env.state).copy()
    ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=horizon, flags=int(auto_reset), n_threads=4)
    d_acts = torch.from_numpy(acts).cuda()
    split = 40
    for t in range(split):
        out = env.step(d_acts[t])
        for got, want in zip(out, ref):
            assert np.array_equal(_np(got), want[t]), t
    out = env.rollout(d_acts[split:].contiguous())
    for got, want in zip(out, ref):
        assert np.array_equal(_np(got), want[split:])
    assert np.array_equal(_np(env.state), ref_state)
    if not auto_reset:  # finished envs are frozen and flagged
        assert (ref[3][-1] == L.EVF_STEPPED_DONE).all() and (ref_state[:, 0] == horizon).all()


@pytest.mark.parametrize("name,S", [("marshmallow_experiment", 64), ("corridor", 128), ("mdp_test", 16)])
def test_wide_records_vs_oracle(name, S):
    n, T = 700, 120
    env = BatchedOvercookedEnv(name, n, horizon=100, auto_reset=True)
    assert env.state_words == S
    rng = np.random.RandomState(S)
    acts = _random_actions(rng, T, n, 0.35)
    ref_state = _np(env.state).copy()
    ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=100, flags=1, n_threads=4)
    out = env.rollout(torch.from_numpy(acts).cuda())
    for got, want in zip(out, ref):
        assert np.array_equal(_np(got), want)
    assert np.array_equal(_np(env.state), ref_state)
    l = env.layouts[0]
    enc = env.lossless_state_encoding(dtype=torch.float32)
    assert np.array_equal(_np(enc), cpu.encode_lossless(env._tab_host, ref_state, l.width, l.height, 100).astype(np.float32))
    f = _np(env.featurize_state(num_pots=2))
    assert np.array_equal(f.astype(np.float64), cpu.featurize(env._tab_host, lut_bytes([l]), ref_state, 2))


def test_mixed_layout_observations_vs_oracle():
    n = 5 * 600 + 1
    env = BatchedOvercookedEnv(CLASSIC5, n, horizon=400, auto_reset=True)
    rng = np.random.RandomState(3)
    env.rollout(torch.from_numpy(_random_actions(rng, 380, n, 0.4)).cuda())
    st = _np(env.state)
    encs = env.lossless_state_encoding(dtype=torch.uint8)
    assert len(encs) == 5
    for (b, e, li), enc in zip(env.segments(), encs):
        l = env.layouts[li]
        want = cpu.encode_lossless(env._tab_host, st[b:e], l.width, l.height, 400)
        assert np.array_equal(_np(enc).astype(np.int32), want)
    f = _np(env.featurize_state(num_pots=2))
    assert np.array_equal(f.astype(np.float64), cpu.featurize(env._tab_host, lut_bytes(env.layouts), st, 2))


def _full_size_check(layouts, n, T, horizon, chunk, seed):
    """BASELINE-size run, compared in full with the (multi-threaded) oracle, chunk by chunk."""
    env = BatchedOvercookedEnv(layouts, n, horizon=horizon, auto_reset=True)
    rng = np.random.RandomState(seed)
    ref_state = _np(env.state).copy()
    tot_sparse = 0
    for c0 in range(0, T, chunk):
        tc = min(chunk, T - c0)
        acts = _random_actions(rng, tc, n, 0.25)
        ref = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=horizon, flags=1, n_threads=0)
        out = env.rollout(torch.from_numpy(acts).cuda())
        for got, want in zip(out, ref):
            assert np.array_equal(_np(got), want)
        tot_sparse += int(ref[0].sum())
    assert np.array_equal(_np(env.state), ref_state)
    # size-independent properties: every env has run the same number of transitions; the horizon
    # was crossed exactly floor(T / horizon) times
    assert (ref_state[:, 0] == T % horizon).all()
    return env, ref_state, tot_sparse


def test_config2_cramped_room_65536_envs_400_steps():
    env, st, _ = _full_size_check("cramped_room", 65536, 400, 400, 50, seed=11)
    assert np.array_equal(st, np.repeat(env._starts_host, 65536, 0))  # all auto-reset to the start record


def test_config3_mixed_5_layouts_262144_envs():
    _full_size_check(CLASSIC5, 262144, 120, 400, 24, seed=12)


def test_config4_asymmetric_advantages_one_shard_of_8():
    _full_size_check("asymmetric_advantages", 1048576 // 8, 200, 400, 40, seed=13)


def test_reset_mask_and_noop_properties():
    n = 3000
    env = BatchedOvercookedEnv(CLASSIC5, n, horizon=400)
    rng = np.random.RandomState(5)
    env.rollout(torch.from_numpy(_random_actions(rng, 50, n)).cuda())
    before = _np(env.state).copy()
    # STAY/STAY only advances the clock and the pots
    stay = torch.full((n, 2), 4, dtype=torch.int32, device="cuda")
    sp, sh, dn, ev = env.step(stay)
    after = _np(env.state)
    assert (after[:, 0] == before[:, 0] + 1).all() and np.array_equal(after[:, 1:4], before[:, 1:4])
    assert not _np(sp).any() and not _np(sh).any() and not _np(ev).any()
    # masked reset touches exactly the masked envs, and is idempotent
    mask = torch.from_numpy((rng.rand(n) < 0.5).astype(np.int32)).cuda()
    env.reset(mask)
    once = _np(env.state).copy()
    env.reset(mask)
    assert np.array_equal(_np(env.state), once)
    m = _np(mask).astype(bool)
    assert np.array_equal(once[~m], after[~m])
    assert np.array_equal(once[m], env._starts_host[env.env_layout_host[m]])
    # determinism: same state + same actions -> same everything
    a = torch.from_numpy(_random_actions(rng, 1, n)[0]).cuda()
    s0 = env.state.clone()
    o1 = [x.clone() for x in env.step(a)]
    s1 = env.state.clone()
    env.state.copy_(s0)
    o2 = env.step(a)
    assert torch.equal(env.state, s1) and all(torch.equal(x, y) for x, y in zip(o1, o2))


@pytest.mark.parametrize("pdl", [False, True], ids=["plain", "pdl"])
def test_cuda_graph_capture_of_step(pdl):
    """The C ABI launches on torch's current stream, so a step can be captured in a CUDA graph
    (also with programmatic dependent launch between consecutive transitions)."""
    n = 4096
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400, auto_reset=True, pdl=pdl)
    ref_env = BatchedOvercookedEnv("cramped_room", n, horizon=400, auto_reset=True)
    rng = np.random.RandomState(9)
    acts = torch.from_numpy(_random_actions(rng, 20, n)).cuda()
    static_a = acts[0].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        env.step(static_a)  # warm up outside capture
    torch.cuda.current_stream().wait_stream(s)
    env.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.step(static_a)
    env.reset()
    for t in range(20):
        static_a.copy_(acts[t])
        g.replay()
        ref_env.step(acts[t])
        assert torch.equal(env.state, ref_env.state) and torch.equal(env.sparse, ref_env.sparse)
        assert torch.equal(env.shaped, ref_env.shaped) and torch.equal(env.events, ref_env.events)
    # a whole episode of back-to-back transitions in ONE graph (the bench's "graph" mode)
    T = 60
    seq = torch.from_numpy(_random_actions(rng, T, n)).cuda()
    outs = [tuple(torch.empty_like(x) for x in (env.sparse, env.shaped, env.done, env.events)) for _ in range(T)]
    env.reset(), ref_env.reset()
    torch.cuda.synchronize()
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        for t in range(T):
            env.step(seq[t], out=outs[t])
    env.reset()
    g2.replay()
    want = ref_env.rollout(seq)
    for t in range(T):
        for got, w in zip(outs[t], want):
            assert torch.equal(got, w[t])
    assert torch.equal(env.state, ref_env.state)


def test_bad_arguments_are_reported():
    lib = _native.lib()
    env = BatchedOvercookedEnv("cramped_room", 8)
    rc = lib.ovc_step(env.tables.data_ptr(), 1, env.start_records.data_ptr(), env.state.data_ptr(), 0, 0, 0, 0, 0, 8, 16, 400, 0, None, 0)
    assert rc == -1 and b"null" in lib.ovc_last_error()
    rc = lib.ovc_step(env.tables.data_ptr(), 1, env.start_records.data_ptr(), env.state.data_ptr(), env.state.data_ptr(),
                      env.sparse.data_ptr(), env.shaped.data_ptr(), env.done.data_ptr(), env.events.data_ptr(), 8, 24, 400, 0, None, 0)
    assert rc == -1 and b"state_words" in lib.ovc_last_error()


def test_selfplay_policy_rollout_matches_oracle_replay():
    """Config-5 pipeline (K2 -> torch CNN -> multinomial -> K1): whatever the policy samples, the
    environments must follow the oracle on those very actions; graph replay == eager."""
    from overcooked_ai_b200.selfplay import SelfPlayRollout

    n, T = 512, 25
    torch.manual_seed(0)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=20, auto_reset=True)
    sp = SelfPlayRollout(env, use_graph=False, autocast_dtype=None)
    ref_state = _np(env.state).copy()
    for t in range(T):
        sp.run(1)
        a = _np(sp.actions)
        assert a.min() >= 0 and a.max() <= 5
        cpu.step(env._tab_host, env._starts_host, ref_state, a, horizon=20, flags=1)
        assert np.array_equal(_np(env.state), ref_state), t
    env2 = BatchedOvercookedEnv("cramped_room", n, horizon=20, auto_reset=True)
    sp2 = SelfPlayRollout(env2, model=sp.model, use_graph=True)
    assert sp2.run(30) == 30 * n and (_np(env2.state)[:, 0] == 30 % 20).all()


def _k7_reference(obs, wt, bias, slope):
    """float64 restatement of ovc_encode_linear on a materialised observation: leaky_relu(obs @ wt + bias)."""
    z = obs.reshape(obs.shape[0] * 2, -1).astype(np.float64) @ wt.astype(np.float64) + bias.astype(np.float64)
    return np.where(z > 0, z, z * slope)


def _k7_close(got, want):
    # bf16 output (8 significant bits, round to nearest) of a float32 accumulation
    return np.abs(got - want) <= np.abs(want) * 2.0 ** -8 + 1e-4


@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_k7_encode_linear_vs_reference_encoding(path):
    """K7 (first layer evaluated from the packed record) against W . (the REFERENCE's lossless_state_encoding, from the
    fixtures) on every layout's trace states: held soups, idle / cooking / ready pots, objects on counters."""
    tr = Trace(path)
    d = tr.data
    st = d["obs_states"]
    W, H = tr.layout.width, tr.layout.height
    env = _env_for_trace(tr, len(st), 0, horizon=400)
    env.state.copy_(torch.from_numpy(st))
    rng = np.random.RandomState(W * 31 + H)
    for n_out, slope in ((64, 0.2), (256, 0.0), (512, 0.2)):
        wt = torch.from_numpy(rng.uniform(-0.05, 0.05, size=(W * H * 26, n_out)).astype(np.float32)).cuda().to(torch.bfloat16)
        bias = torch.from_numpy(rng.uniform(-0.1, 0.1, size=n_out).astype(np.float32)).cuda()
        if W * H * 19 * 64 * 2 > 226 * 1024:  # the table of this grid does not fit shared memory: refused, not wrong
            with pytest.raises(RuntimeError, match="shared memory"):
                env.encoded_linear(wt, bias, neg_slope=slope)
            continue
        got = _np(env.encoded_linear(wt, bias, neg_slope=slope).float())
        want = _k7_reference(d["obs_lossless"], _np(wt.float()), _np(bias), slope)
        assert got.shape == want.shape and _k7_close(got, want).all(), (n_out, np.abs(got - want).max())


def test_k7_encode_linear_views_urgency_layout_mix_and_ragged_sizes():
    """view_swap, the urgency plane (horizon - t < 40), two layouts of one grid shape in one call, batch sizes that are not
    multiples of a warp / the CTA's warps: K7 == W . K2 (K2 itself is tested against the reference's encoding)."""
    rng = np.random.RandomState(5)
    for layouts, n, horizon in ((["cramped_room", "cramped_room_tomato"], 2 * 333 + 1, 60), (["asymmetric_advantages"], 1027, 60),
                                (["cramped_room"], 1, 400)):
        env = BatchedOvercookedEnv(layouts, n, horizon=horizon, auto_reset=True)
        env.rollout(torch.from_numpy(_random_actions(rng, 30, n, 0.5)).cuda())
        env.reset(torch.from_numpy((rng.rand(n) < 0.5).astype(np.int32)).cuda())  # half of them start over: timesteps 15 and 45
        env.rollout(torch.from_numpy(_random_actions(rng, 15, n, 0.5)).cuda())
        W, H = env.layouts[0].width, env.layouts[0].height
        wt = torch.from_numpy(rng.uniform(-0.05, 0.05, size=(W * H * 26, 128)).astype(np.float32)).cuda().to(torch.bfloat16)
        bias = torch.from_numpy(rng.uniform(-0.1, 0.1, size=128).astype(np.float32)).cuda()
        swap = torch.from_numpy((rng.rand(n) < 0.5).astype(np.int32)).cuda()
        for vs in (None, swap):
            obs = _np(env.lossless_state_encoding(dtype=torch.float32, view_swap=vs))
            assert n == 1 or (obs[..., 25].any() and not obs[..., 25].all())  # some environments are in their last 40 steps
            got = _np(env.encoded_linear(wt, bias, neg_slope=0.3, view_swap=vs).float())
            want = _k7_reference(obs, _np(wt.float()), _np(bias), 0.3)
            assert _k7_close(got, want).all(), np.abs(got - want).max()
    lib = _native.lib()
    rc = lib.ovc_encode_linear(env.tables.data_ptr(), 1, env.state.data_ptr(), 0, wt.data_ptr(), bias.data_ptr(), wt.data_ptr(), 1, 16, 5, 4,
                               400, 100, 0.2, 0)
    assert rc == -1 and b"multiple of 64" in lib.ovc_last_error()


def test_selfplay_fused_first_layer_equals_unfused_policy():
    """Config 5 with K7 in front of the dense policy == the same policy on K2's observation tensor (same weights; bf16
    activations, so logits agree to bf16 accuracy), and the environments follow the oracle on the sampled actions."""
    from overcooked_ai_b200.selfplay import SelfPlayRollout

    n = 777
    torch.manual_seed(3)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=30, auto_reset=True)
    rng = np.random.RandomState(9)
    env.rollout(torch.from_numpy(_random_actions(rng, 17, n, 0.5)).cuda())
    fused = SelfPlayRollout(env, use_graph=False, fused_tail=False)
    assert fused.fused_first_layer and fused.obs is None
    plain = SelfPlayRollout(env, model=fused.model, use_graph=False, fused_first_layer=False, fused_tail=False)
    env.lossless_state_encoding(out=plain.obs)
    a, b = _np(fused._policy().clone()), _np(plain._policy().clone())
    assert np.abs(a - b).max() < 0.02 and np.abs(a).max() > 0.01, np.abs(a - b).max()
    # K8 behind K7: the heads it computes are the unfused policy's logits / values; its actions are the draw on them
    tail = SelfPlayRollout(env, model=fused.model, use_graph=False, seed=11)
    assert tail.fused_tail and tail.fused_first_layer and tail.fused_wide
    lib_trunk = SelfPlayRollout(env, model=fused.model, use_graph=False, seed=11, fused_wide=False)
    lib_trunk._policy()
    z_lib = _np(lib_trunk._z.float())
    tail._scores8 = torch.zeros((2 * n, 8), dtype=torch.float32, device="cuda")
    before = _np(env.state).copy()
    assert tail._policy() is None and np.array_equal(_np(env.state), before)
    s8 = _np(tail._scores8)
    assert np.abs(_np(tail._z.float()) - z_lib).max() < 0.05 and np.abs(z_lib).max() > 0.05  # K9 == the two library GEMMs + activation
    assert np.abs(s8[:, :6] - b).max() < 0.02 and np.abs(s8[:, 6] - _np(plain.values).reshape(-1)).max() < 0.02
    assert np.array_equal(s8[:, 6], _np(tail.values).reshape(-1)) and _np(tail._draw_counter).tolist() == [1, 0]
    assert _np(lib_trunk._draw_counter).tolist() == [1, 0]
    _check_draw(_np(tail.actions).reshape(-1), s8, 11, 0)
    ref_state = _np(env.state).copy()
    for t in range(20):
        fused.run(1)
        cpu.step(env._tab_host, env._starts_host, ref_state, _np(fused.actions), horizon=30, flags=1)
        assert np.array_equal(_np(env.state), ref_state), t
    g = SelfPlayRollout(env, model=fused.model, use_graph=True)
    assert g.run(12) == 12 * n


def _philox4x32_10(key, c):
    """numpy restatement of Philox4x32-10 (Salmon et al.): key uint64, c uint32[n, 4] -> uint32[n, 4]."""
    c = [c[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key & 0xFFFFFFFF), np.uint64(key >> 32)
    M = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return np.stack(c, 1).astype(np.uint32)


def test_sample_actions_kernel_matches_its_definition_and_softmax():
    """ovc_sample_actions: the draw is the documented function of (seed, step, row) — numpy restatement of the Philox
    counter plan and the Gumbel-max rule; the step advances by one per launch; frequencies follow softmax(logits)."""
    n = 40000
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400)
    rng = np.random.RandomState(2)
    scores = torch.from_numpy(rng.normal(size=(2 * n, 8)).astype(np.float32)).cuda()
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    seed = 0x1234567890ABCDEF
    rows = np.arange(2 * n, dtype=np.uint64)
    freq = np.zeros(6)
    for step in range(3):
        a = _np(env.sample_actions(scores, counter, seed=seed)).reshape(-1)
        assert _np(counter).tolist() == [step + 1, 0]
        ctr = np.stack([rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32), np.full_like(rows, step), np.zeros_like(rows)], 1).astype(np.uint32)
        d = np.concatenate([_philox4x32_10(seed, ctr), _philox4x32_10(seed, ctr | np.array([0, 0, 0, 1], np.uint32))], 1)[:, :6]
        u = ((d >> np.uint32(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
        v = _np(scores)[:, :6] - np.log(-np.log(u))
        want = v.argmax(1)
        top2 = np.sort(v, 1)[:, -2:]
        clear = top2[:, 1] - top2[:, 0] > 1e-4  # libm and the device logf differ in the last bits: near-ties may flip
        assert clear.mean() > 0.999 and np.array_equal(a[clear], want[clear])
        assert a.min() >= 0 and a.max() <= 5
        freq += np.bincount(a, minlength=6)
    # one fixed logit row for everybody: empirical frequencies == softmax within sampling error
    scores[:] = torch.tensor([0.5, -1.0, 2.0, 0.0, 1.0, -0.5, 99.0, 99.0], device="cuda")
    a = np.concatenate([_np(env.sample_actions(scores, counter, seed=7)).reshape(-1) for _ in range(5)])
    p = np.exp([0.5, -1.0, 2.0, 0.0, 1.0, -0.5])
    p /= p.sum()
    f = np.bincount(a, minlength=6) / a.size
    assert np.abs(f - p).max() < 4 * np.sqrt(0.25 / a.size), (f, p)


@pytest.mark.parametrize("layout,flags", [("coordination_ring", (True, False, False)), ("asymmetric_advantages", (False, False, False))])
def test_selfplay_other_grids_fall_back_to_library_layers(layout, flags):
    """Grids whose policy widths the fused kernels are not built for (5x5: K7 only; 9x5: none) run the remaining layers as
    library GEMMs with the separate draw kernel; the environments still follow the oracle on the drawn actions."""
    from overcooked_ai_b200.selfplay import SelfPlayRollout

    n = 300
    torch.manual_seed(1)
    env = BatchedOvercookedEnv(layout, n, horizon=25, auto_reset=True)
    sp = SelfPlayRollout(env, use_graph=False, seed=2)
    assert (sp.fused_first_layer, sp.fused_wide, sp.fused_tail) == flags and sp.native_glue
    ref_state = _np(env.state).copy()
    for t in range(30):
        sp.run(1)
        a = _np(sp.actions)
        assert a.min() >= 0 and a.max() <= 5
        cpu.step(env._tab_host, env._starts_host, ref_state, a, horizon=25, flags=1)
        assert np.array_equal(_np(env.state), ref_state), t
    assert len(np.unique(_np(sp.actions))) > 3


def _check_draw(actions, scores, seed, step, n_actions=6):
    """actions == the ovc_sample_actions definition applied to ``scores`` (numpy restatement; near-ties exempt)."""
    rows = np.arange(len(scores), dtype=np.uint64)
    ctr = np.stack([rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32), np.full_like(rows, step), np.zeros_like(rows)], 1).astype(np.uint32)
    d = np.concatenate([_philox4x32_10(seed, ctr), _philox4x32_10(seed, ctr | np.array([0, 0, 0, 1], np.uint32))], 1)[:, :n_actions]
    u = ((d >> np.uint32(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    v = scores[:, :n_actions] - np.log(-np.log(u))
    top2 = np.sort(v, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-4  # libm and the device logf differ in the last bits: near-ties may flip
    assert clear.mean() > 0.995 and np.array_equal(actions[clear], v.argmax(1)[clear])
    assert actions.min() >= 0 and actions.max() < n_actions


def _bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float().numpy()


@pytest.mark.parametrize("k0,n_hidden,n_rows", [(160, 2, 4099), (64, 0, 16), (256, 3, 1000), (96, 1, 1)])
def test_k8_policy_tail_vs_float_reference(k0, n_hidden, n_rows):
    """K8 (dense tail + heads + draw in one kernel) against a float32 restatement with bf16 rounding between layers; the
    actions are the documented draw on the heads the kernel itself reports; ragged row counts; the step advances."""
    lib = _native.lib()
    rng = np.random.RandomState(k0 + n_hidden)
    x = _bf16(rng.normal(size=(n_rows, k0)))
    w1, b1 = _bf16(rng.normal(size=(64, k0)) / np.sqrt(k0)), rng.normal(size=64).astype(np.float32) * 0.1
    wh, bh = _bf16(rng.normal(size=(max(n_hidden, 1), 64, 64)) / 8), rng.normal(size=(max(n_hidden, 1), 64)).astype(np.float32) * 0.1
    wo, bo = _bf16(rng.normal(size=(8, 64)) / 4), rng.normal(size=8).astype(np.float32) * 0.1
    lrelu = lambda z, s: np.where(z > 0, z, z * np.float32(s)).astype(np.float32)
    a = _bf16(lrelu(x, 0.2))
    a = _bf16(lrelu(a @ w1.T + b1, 0.3))
    for l in range(n_hidden):
        a = _bf16(lrelu(a @ wh[l].T + bh[l], 0.3))
    want = a @ wo.T + bo
    dev = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)
    tx, tw1, twh, two = dev(x, torch.bfloat16), dev(w1, torch.bfloat16), dev(wh, torch.bfloat16), dev(wo, torch.bfloat16)
    tb1, tbh, tbo = dev(b1, torch.float32), dev(bh, torch.float32), dev(bo, torch.float32)
    counter = torch.zeros(2, dtype=torch.int64, device="cuda")
    actions = torch.full((n_rows,), -1, dtype=torch.int32, device="cuda")
    values = torch.zeros(n_rows, dtype=torch.float32, device="cuda")
    scores = torch.zeros((n_rows, 8), dtype=torch.float32, device="cuda")
    for step in range(2):
        _native.check(lib.ovc_policy_tail(tx.data_ptr(), n_rows, k0, 0.2, tw1.data_ptr(), tb1.data_ptr(), twh.data_ptr(), tbh.data_ptr(), n_hidden,
                                          two.data_ptr(), tbo.data_ptr(), 0.3, 6, 99, counter.data_ptr(), actions.data_ptr(), values.data_ptr(),
                                          scores.data_ptr(), 0))
        got = _np(scores)
        assert np.abs(got - want).max() < 0.03 * max(1.0, np.abs(want).max()), np.abs(got - want).max()
        assert np.array_equal(_np(values), got[:, 6]) and _np(counter).tolist() == [step + 1, 0]
        if n_rows >= 1000:
            _check_draw(_np(actions), got, 99, step)
        else:
            assert _np(actions).min() >= 0 and _np(actions).max() <= 5
    rc = lib.ovc_policy_tail(tx.data_ptr(), n_rows, 100, 0.2, tw1.data_ptr(), tb1.data_ptr(), twh.data_ptr(), tbh.data_ptr(), n_hidden,
                             two.data_ptr(), tbo.data_ptr(), 0.3, 6, 99, counter.data_ptr(), actions.data_ptr(), 0, 0, 0)
    assert rc == -1 and b"multiple of 32" in lib.ovc_last_error()


@pytest.mark.parametrize("m", [128, 1000, 1, 4096 + 77, 128 * 449 + 5])
def test_k9_wide_layers_vs_float_reference(m):
    """K9 (wgmma: a1 = leaky_relu(a0 W1^T + b1) kept in registers, z2 = a1 W2^T + b2) against a float32 restatement with the
    activation rounded to bf16 between the layers; partial last tiles; the largest case gives every persistent CTA three or
    four tiles (barrier phases, accumulator and shared-memory re-use across tiles)."""
    lib = _native.lib()
    rng = np.random.RandomState(m)
    a0 = _bf16(rng.normal(size=(m, 512)))
    w1, b1 = _bf16(rng.normal(size=(512, 512)) / np.sqrt(512)), rng.normal(size=512).astype(np.float32) * 0.2
    w2, b2 = _bf16(rng.normal(size=(160, 512)) / np.sqrt(512)), rng.normal(size=160).astype(np.float32) * 0.2
    z1 = a0 @ w1.T + b1
    a1 = _bf16(np.where(z1 > 0, z1, z1 * np.float32(0.2)))
    want = a1 @ w2.T + b2
    dev = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)
    ta0, tw1, tw2 = dev(a0, torch.bfloat16), dev(w1, torch.bfloat16), dev(w2, torch.bfloat16)
    tb1, tb2 = dev(b1, torch.float32), dev(b2, torch.float32)
    z2 = torch.full((m, 160), float("nan"), dtype=torch.bfloat16, device="cuda")
    _native.check(lib.ovc_wide_layers(ta0.data_ptr(), m, 512, tw1.data_ptr(), tb1.data_ptr(), 512, tw2.data_ptr(), tb2.data_ptr(), 160, 0.2,
                                      z2.data_ptr(), 0))
    torch.cuda.synchronize()
    got = _np(z2.float())
    assert np.isfinite(got).all()
    err = np.abs(got - want)
    assert (err <= np.abs(want) * 2.0 ** -7 + 0.02).all(), (err.max(), np.abs(want).max())
    rc = lib.ovc_wide_layers(ta0.data_ptr(), m, 256, tw1.data_ptr(), tb1.data_ptr(), 512, tw2.data_ptr(), tb2.data_ptr(), 160, 0.2, z2.data_ptr(), 0)
    assert rc == -3 and b"512 -> 512 -> 160" in lib.ovc_last_error()


def test_accumulate_returns_kernel():
    n = 3001
    env = BatchedOvercookedEnv("cramped_room", n, horizon=400, auto_reset=True)
    rng = np.random.RandomState(4)
    rs, rm = torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.float32, device="cuda")
    ws, wm = np.zeros(n, np.int64), np.zeros(n, np.float64)
    for t in range(120):
        sp, sh, dn, ev = env.step(torch.from_numpy(_random_actions(rng, 1, n, 0.6)[0]).cuda())
        env.accumulate_returns(rs, rm, 0.75)
        ws += _np(sp)
        wm += _np(sp) + 0.75 * _np(sh).sum(1)
    assert ws.sum() >= 0 and wm.max() > 0 and np.array_equal(_np(rs), ws) and np.allclose(_np(rm), wm, rtol=1e-6, atol=1e-4)


@pytest.mark.parametrize("gamma_idx,gamma", [(0, 0.99), (1, 0.9)])
def test_potential_kernel_bit_exact_vs_reference(gamma_idx, gamma):
    """K6: phi(s) equals the reference's potential_function float for float (fixture from the reference)."""
    g = np.load(GOLD + "/potential.npz")
    for path in TRACE_FILES:
        name = path.split("trace_")[-1][:-4]
        if name + "__phi" not in g.files:
            continue
        tr = Trace(path)
        st = tr.data["obs_states"]
        env = _env_for_trace(tr, len(st), 0)
        env.state.copy_(torch.from_numpy(st))
        phi = _np(env.potential(gamma))
        assert phi.dtype == np.float64 and np.array_equal(phi, g[name + "__phi"][:, gamma_idx]), name


def test_potential_kernel_vs_oracle_mixed_layouts():
    n = 5 * 4000 + 7
    env = BatchedOvercookedEnv(CLASSIC5, n, horizon=400, auto_reset=True)
    rng = np.random.RandomState(21)
    env.rollout(torch.from_numpy(_random_actions(rng, 150, n, 0.45)).cuda())
    st = _np(env.state)
    pt, cst, gpow = L.build_potential_tables(env.layouts, 0.99)
    want = cpu.potential(env._tab_host, pt, cst, gpow, st)
    got = _np(env.potential(0.99))
    assert np.array_equal(got, want) and len(np.unique(got)) > 50


def test_narrow_transfer_formats_and_host_pipeline():
    """uint8 actions in / int16-int8-uint8 outputs: the same values as the int32 formats; the host pipeline
    (pinned host buffers, chunked, three streams) equals one device-side rollout."""
    from overcooked_ai_b200.batched import HostRolloutPipeline

    n, T = 3001, 130
    rng = np.random.RandomState(31)
    acts = _random_actions(rng, T, n, 0.4)
    env_a = BatchedOvercookedEnv("cramped_room", n, horizon=50, auto_reset=True)
    env_b = BatchedOvercookedEnv("cramped_room", n, horizon=50, auto_reset=True)
    assert env_a.narrow_ok()
    want = env_a.rollout(torch.from_numpy(acts).cuda())
    from overcooked_ai_b200 import wire

    env_b.reset()
    pipe = HostRolloutPipeline(env_b, T, chunk=32, packed=True)
    got = pipe.run(torch.from_numpy(acts.astype(np.uint8)).pin_memory())
    torch.cuda.synchronize()
    assert got[2] is None and got[3].dtype == torch.int16 and pipe.d2h_bytes_per_step == n * 6
    ev, dn = wire.decode_event_codes(got[3].numpy())
    assert np.array_equal(got[0].numpy(), _np(want[0])) and np.array_equal(got[1].numpy(), _np(want[1]))
    assert np.array_equal(ev, _np(want[3])) and np.array_equal(dn, _np(want[2]) != 0)
    assert torch.equal(env_b.state, env_a.state)
    for narrow in (True, False):
        env_b.reset()
        pipe = HostRolloutPipeline(env_b, T, chunk=32, narrow=narrow)
        h_act = torch.from_numpy(acts.astype(np.uint8 if narrow else np.int32)).pin_memory()
        got = pipe.run(h_act)
        torch.cuda.synchronize()
        assert got[0].dtype == (torch.int16 if narrow else torch.int32) and got[0].is_pinned()
        for g, w in zip(got, want):
            assert np.array_equal(g.numpy().astype(np.int64), _np(w).astype(np.int64))
        assert torch.equal(env_b.state, env_a.state)


def test_code_words_and_one_byte_actions_carry_the_whole_result():
    """OVC_F_OUT_CODES / OVC_F_ACT_PACKED: 1 byte in, 2 bytes out per env-step; expanding the words on the host
    gives back sparse / shaped / done / events of the int32 formats, through rollout() and the host pipeline."""
    from overcooked_ai_b200 import wire

    n, T = 6007, 96
    names = ["cramped_room", "counter_circuit", "asymmetric_advantages"]
    rng = np.random.RandomState(4)
    acts = _random_actions(rng, T, n, 0.45)
    env_a = BatchedOvercookedEnv(names, n, horizon=40, auto_reset=True, rnd_obj_prob_thresh=0.6, seed=9)
    env_b = BatchedOvercookedEnv(names, n, horizon=40, auto_reset=True, rnd_obj_prob_thresh=0.6, seed=9)
    want = [_np(x) for x in env_a.rollout(torch.from_numpy(acts).cuda())]
    assert want[0].max() >= 20 and (want[1] > 0).any() and (want[3] & (1 << 14)).any()
    packed_acts = wire.pack_actions(acts)
    out = env_b.alloc_rollout_out(T, codes=True)
    env_b.rollout(torch.from_numpy(packed_acts).cuda(), out=out)
    assert out[0] is None and torch.equal(env_b.state, env_a.state)
    words = out[3].cpu()
    got = wire.decode_codes(words.numpy(), env_b.code_reward_table(), env_b.env_layout_host)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(got[2], want[2] != 0) and np.array_equal(got[3], want[3])
    dense = env_b.expand_codes(words, events=True)
    assert np.array_equal(dense["sparse"].numpy(), want[0]) and np.array_equal(dense["shaped"].numpy(), want[1])
    assert np.array_equal(dense["done"].numpy(), want[2]) and np.array_equal(dense["events"].numpy(), want[3])
    # the dish / soup taken from a counter logs the pickup event but grants nothing: the case the grant bits exist for
    ev, sh = want[3], want[1]
    assert ((ev & (1 << 14)) != 0)[sh == 0].any() and ((ev & (1 << 14)) != 0)[sh == 5].any()
    env_b.reset()
    env_a.reset()
    want = [_np(x) for x in env_a.rollout(torch.from_numpy(acts).cuda())]
    pipe = HostRolloutPipeline(env_b, T, chunk=40, codes=True)
    assert pipe.h2d_bytes_per_step == n and pipe.d2h_bytes_per_step == 2 * n
    h = pipe.run(torch.from_numpy(packed_acts).pin_memory())
    torch.cuda.synchronize()
    dense = env_b.expand_codes(h[3], events=True)
    assert np.array_equal(dense["sparse"].numpy(), want[0]) and np.array_equal(dense["shaped"].numpy(), want[1])
    assert np.array_equal(dense["done"].numpy(), want[2]) and np.array_equal(dense["events"].numpy(), want[3])
    assert torch.equal(env_b.state, env_a.state)
    # two passes submitted back to back without joining the current stream in between (two pinned output sets)
    want2 = [_np(x) for x in env_a.rollout(torch.from_numpy(acts[::-1].copy()).cuda())]
    want3 = [_np(x) for x in env_a.rollout(torch.from_numpy(acts).cuda())]
    pipe = HostRolloutPipeline(env_b, T, chunk=40, codes=True, host_buffers=2)
    rev = torch.from_numpy(wire.pack_actions(acts[::-1])).pin_memory()
    fwd = torch.from_numpy(packed_acts).pin_memory()
    (h2, e2), (h3, e3) = pipe.run(rev, wait=False), pipe.run(fwd, wait=False)
    assert h2[3].data_ptr() != h3[3].data_ptr()
    for h, e, w in ((h2, e2, want2), (h3, e3, want3)):
        e.synchronize()
        dense = env_b.expand_codes(h[3], events=True)
        assert np.array_equal(dense["sparse"].numpy(), w[0]) and np.array_equal(dense["shaped"].numpy(), w[1])
        assert np.array_equal(dense["done"].numpy(), w[2]) and np.array_equal(dense["events"].numpy(), w[3])
    pipe.join()
    assert torch.equal(env_b.state, env_a.state)


def test_sparse_event_stream_carries_the_whole_result():
    """OVC_F_OUT_STREAM: one warp vote (lane mask) per 32 environments and transition + the compacted non-zero code
    words.  Expanded on the host it must give back sparse / shaped / done / events of the int32 formats — through
    rollout_stream() (partial last group, random-start auto-resets, mixed layouts, stepped-after-done words) and through
    the host pipeline; a capacity that is too small is counted, and the dense backup recovers the pass."""
    from overcooked_ai_b200 import wire

    n, T = 6007, 96  # 6007 = 187 full groups + one of 23 environments
    names = ["cramped_room", "counter_circuit", "asymmetric_advantages"]
    rng = np.random.RandomState(4)
    acts = _random_actions(rng, T, n, 0.45)
    kw = dict(horizon=40, auto_reset=True, rnd_obj_prob_thresh=0.6, seed=9)
    env_a, env_b = BatchedOvercookedEnv(names, n, **kw), BatchedOvercookedEnv(names, n, **kw)
    want = [_np(x) for x in env_a.rollout(torch.from_numpy(acts).cuda())]
    masks, values, dense_words = env_b.rollout_stream(torch.from_numpy(wire.pack_actions(acts)).cuda(), cap=T * 32, dense_backup=True)
    assert torch.equal(env_b.state, env_a.state)
    env_c = BatchedOvercookedEnv(names, n, **kw)  # a third copy of the same start states for the dense code words
    codes = env_c.alloc_rollout_out(T, codes=True)
    env_c.rollout(torch.from_numpy(wire.pack_actions(acts)).cuda(), out=codes)
    assert torch.equal(dense_words, codes[3]), "the dense backup is the OVC_F_OUT_CODES word"
    nz = _np(codes[3]) != 0
    m = _np(masks).view(np.uint32)
    bits = ((m[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(T, -1)[:, :n].astype(bool)
    assert np.array_equal(bits, nz) and 0.02 < nz.mean() < 0.5, "lane masks = non-zero words"
    got, over = env_b.expand_stream(masks.cpu(), values.cpu(), events=True)
    assert over == 0
    for k, w in zip(("sparse", "shaped", "done", "events"), want):
        assert np.array_equal(got[k].numpy(), w), k
    # too small a capacity: nothing is written out of bounds, the overflow is counted (a fresh env: the same trajectory)
    env_d = BatchedOvercookedEnv(names, n, **kw)
    G = env_d.n_groups()
    per_group = np.pad(bits, ((0, 0), (0, G * 32 - n))).reshape(T, G, 32).sum((0, 2))
    cap = int(per_group.max()) - 1
    guard = torch.full((G * cap + 64,), 0x5A5A, dtype=torch.int16, device="cuda")
    out = (torch.zeros((T, G), dtype=torch.int32, device="cuda"), guard[: G * cap].view(1, G, cap), None)
    env_d.rollout_stream(torch.from_numpy(acts).cuda(), cap=cap, out=out)
    assert (guard[G * cap:] == 0x5A5A).all() and torch.equal(env_d.state, env_a.state)
    _, over = env_d.expand_stream(out[0].cpu(), out[1].cpu().contiguous())
    assert over == int((per_group > cap).sum()) >= 1
    # ---- the host pipeline: chunks, two overlapping passes, and an overflow recovered from the device-side backup ----
    env_e, env_f = BatchedOvercookedEnv(names, n, **kw), BatchedOvercookedEnv(names, n, **kw)
    want1 = [_np(x) for x in env_e.rollout(torch.from_numpy(acts).cuda())]
    want2 = [_np(x) for x in env_e.rollout(torch.from_numpy(acts[::-1].copy()).cuda())]
    pipe = HostRolloutPipeline(env_f, T, chunk=40, stream=True, stream_fill=0.5, host_buffers=2)
    assert pipe.stream_cap == 640 and pipe.h2d_bytes_per_step == n
    fwd, rev = torch.from_numpy(wire.pack_actions(acts)).pin_memory(), torch.from_numpy(wire.pack_actions(acts[::-1])).pin_memory()
    (h1, e1), s1 = pipe.run(fwd, wait=False), pipe._last_set
    (h2, e2), s2 = pipe.run(rev, wait=False), pipe._last_set
    assert s1 != s2
    for h, e, st, w in ((h1, e1, s1, want1), (h2, e2, s2, want2)):
        e.synchronize()
        dense = pipe.expand(h, codes_set=st, events=True)
        assert pipe.last_overflow == 0
        for k, x in zip(("sparse", "shaped", "done", "events"), w):
            assert np.array_equal(dense[k].numpy(), x), k
    pipe.join()
    torch.cuda.synchronize()
    assert torch.equal(env_f.state, env_e.state)
    pipe.close()
    env_g = BatchedOvercookedEnv(names, n, **kw)
    pipe = HostRolloutPipeline(env_g, T, chunk=40, stream=True, stream_fill=0.02, packed_actions=False)  # 26 slots per group and chunk
    h = pipe.run(torch.from_numpy(acts.astype(np.uint8)).pin_memory())
    torch.cuda.synchronize()
    dense = pipe.expand(h, events=True)
    assert pipe.last_overflow > 0, "the capacity was chosen to overflow"
    for k, x in zip(("sparse", "shaped", "done", "events"), want):
        assert np.array_equal(dense[k].numpy(), x), k
    pipe.close()
    # not available where the rollout kernel is not: the per-step record I/O experiments and > 8 layouts
    env_c = BatchedOvercookedEnv("cramped_room", 64, io=_native.IO_DIRECT)
    with pytest.raises(RuntimeError, match="OVC_F_OUT_STREAM"):
        env_c.rollout_stream(torch.zeros((4, 64, 2), dtype=torch.int32, device="cuda"), cap=16)


@pytest.mark.parametrize("random_pos,thresh", [(True, 0.0), (False, 0.7), (True, 0.5)])
def test_random_start_states_vs_oracle_mirror(random_pos, thresh):
    """get_random_start_state_fn on the device (reset + auto-reset inside step / rollout): bit-exact against the
    CPU mirror of the documented generator; episodes differ from each other and between environments."""
    n, horizon, T = 4099, 15, 50
    env = BatchedOvercookedEnv(["cramped_room", "counter_circuit"], n, horizon=horizon, auto_reset=True,
                               random_start_pos=random_pos, rnd_obj_prob_thresh=thresh, seed=77)
    rs = cpu.random_start(77, thresh, random_pos)
    ref = np.zeros((n, env.state_words), np.int32)
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs, env_layout=env.env_layout_host)
    assert np.array_equal(_np(env.state), ref)
    first = ref.copy()
    rng = np.random.RandomState(8)
    acts = _random_actions(rng, T, n, 0.35)
    want = cpu.rollout(env._tab_host, env._starts_host, ref, acts, horizon=horizon, flags=1, n_threads=4, rs=rs)
    d = torch.from_numpy(acts).cuda()
    for t in range(20):
        got = env.step(d[t])
        for g, w in zip(got, want):
            assert np.array_equal(_np(g), w[t]), t
    got = env.rollout(d[20:].contiguous())
    for g, w in zip(got, want):
        assert np.array_equal(_np(g), w[20:])
    assert np.array_equal(_np(env.state), ref)
    assert ((ref[:, 3] >> 16) & 0xFFFF == 1 + T // horizon).all()
    # a masked reset redraws exactly the masked envs, with a new episode number
    mask = (rng.rand(n) < 0.3).astype(np.int32)
    env.reset(torch.from_numpy(mask).cuda())
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs, mask=mask)
    assert np.array_equal(_np(env.state), ref)
    assert len(np.unique(first[:, 1:3], axis=0)) > 10


@pytest.mark.parametrize("pool_size,random_pos,thresh", [(5, False, 0.0), (12, True, 0.4)])
def test_variable_mdp_layout_redraw_vs_oracle_mirror(pool_size, random_pos, thresh):
    """Variable MDP (OvercookedEnv over a LayoutGenerator, overcooked_env.py:288-302): reset and the auto-reset
    inside step / rollout redraw each environment's layout from a pool of generated layouts; bit-exact against
    the CPU mirror, on the shared-memory table path (5 layouts) and the global one (12), observations included."""
    from overcooked_ai_b200 import layout_generator as LG

    np.random.seed(pool_size)
    params = {"inner_shape": (6, 5), "prop_empty": 0.6, "prop_feats": 0.3, "display": False, "feature_types": ["P", "D", "S", "O", "T"],
              "start_all_orders": [{"ingredients": ["onion", "tomato"]}, {"ingredients": ["onion", "onion", "onion"]}]}
    pool = LG.generate_layout_pool(pool_size, params, outer_shape=(7, 6), skip_unsupported=True)
    assert len({tuple("".join(r) for r in l.terrain_mtx) for l in pool}) == pool_size
    n, horizon, T = 3001, 12, 40
    env = BatchedOvercookedEnv(pool, n, horizon=horizon, auto_reset=True, random_layout=True,
                               random_start_pos=random_pos, rnd_obj_prob_thresh=thresh, seed=5)
    rs = cpu.random_start(5, thresh, random_pos, random_layout=True)
    ref = np.zeros((n, env.state_words), np.int32)
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs)
    assert np.array_equal(_np(env.state), ref)
    ids0 = ref[:, 3] & 0xFF
    assert len(np.unique(ids0)) == pool_size and np.array_equal(_np(env.layout_ids()), ids0)
    rng = np.random.RandomState(2)
    acts = _random_actions(rng, T, n, 0.4)
    want = cpu.rollout(env._tab_host, env._starts_host, ref, acts, horizon=horizon, flags=1, n_threads=4, rs=rs)
    d = torch.from_numpy(acts).cuda()
    stats = EpisodeStats(env)
    cum = np.zeros((n, 2), np.int64)
    val = np.stack([l.deliver_value for l in pool])
    lids = ids0.copy()
    for t in range(15):
        got = env.step(d[t])
        for g, w in zip(got, want):
            assert np.array_equal(_np(g), w[t]), t
        ev = want[3][t]
        cum += val[lids[:, None], (ev >> 25) & 15] * ((ev >> 15) & 1)
        fin = stats.update(*got)
        if fin is not None:
            assert np.array_equal(_np(fin["ep_sparse_r_by_agent"]), cum[_np(fin["env_index"])])
            cum[:] = 0
        lids = _np(env.layout_ids()).astype(np.int64)
    got = env.rollout(d[15:].contiguous())
    for g, w in zip(got, want):
        assert np.array_equal(_np(g), w[15:])
    assert np.array_equal(_np(env.state), ref)
    assert ((ref[:, 3] >> 16) & 0xFFFF == 1 + T // horizon).all() and ((ref[:, 3] & 0xFF) != ids0).mean() > 0.5
    # observations of the mixed batch
    W, H = pool[0].width, pool[0].height
    assert np.array_equal(_np(env.lossless_state_encoding(dtype=torch.int32)),
                          cpu.encode_lossless(env._tab_host, ref, W, H, horizon))
    assert np.array_equal(_np(env.featurize_state(2)).astype(np.float64), cpu.featurize(env._tab_host, lut_bytes(pool), ref, 2))
    pt, cst, gpow = L.build_potential_tables(pool, 0.99)
    assert np.array_equal(_np(env.potential(0.99)), cpu.potential(env._tab_host, pt, cst, gpow, ref))
    # masked reset: new layouts for exactly the masked environments
    mask = (rng.rand(n) < 0.5).astype(np.int32)
    env.reset(torch.from_numpy(mask).cuda())
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs, mask=mask)
    assert np.array_equal(_np(env.state), ref)
    # host view of single environments follows the current layout
    s = env.get_states([0, 1, n - 1])
    for k, i in enumerate([0, 1, n - 1]):
        assert s[k].player_positions == tuple((int(ref[i, 1 + j]) & 15, (int(ref[i, 1 + j]) >> 4) & 15) for j in range(2))


def test_more_than_eight_layouts_uses_global_tables():
    """With more than 8 layouts the kernel reads the layout table from global memory instead of staging it in
    shared memory; old_dynamics and new-dynamics layouts mix in one batch."""
    names = ["cramped_room", "asymmetric_advantages", "coordination_ring", "forced_coordination", "counter_circuit",
             "bottleneck", "centre_pots", "random0", "random3", "scenario1_s", "schelling_s"]
    layouts = [L.compile_layout(n) for n in names] + [L.compile_layout("cramped_room", old_dynamics=True)]
    n = len(layouts) * 300 + 5
    env = BatchedOvercookedEnv(layouts, n, horizon=40, auto_reset=True)
    assert env.n_layouts == 12 and env.state_words == 32
    rng = np.random.RandomState(12)
    acts = _random_actions(rng, 100, n, 0.4)
    ref_state = _np(env.state).copy()
    want = cpu.rollout(env._tab_host, env._starts_host, ref_state, acts, horizon=40, flags=1, n_threads=4)
    d = torch.from_numpy(acts).cuda()
    for t in range(30):
        got = env.step(d[t])
        for g, w in zip(got, want):
            assert np.array_equal(_np(g), w[t]), t
    got = env.rollout(d[30:].contiguous())
    for g, w in zip(got, want):
        assert np.array_equal(_np(g), w[30:])
    assert np.array_equal(_np(env.state), ref_state)
    f = _np(env.featurize_state(2))
    assert np.array_equal(f.astype(np.float64), cpu.featurize(env._tab_host, lut_bytes(env.layouts), ref_state, 2))


def _all_two_player_layouts():
    out = []
    for n in L.layout_names():
        try:
            L.compile_layout(n)
            out.append(n)
        except ValueError:
            pass
    return out


@pytest.mark.parametrize("name", _all_two_player_layouts())
def test_every_bundled_layout_vs_oracle(name):
    """All 44 bundled 2-player layouts: random start states, 90 transitions across a horizon, every output,
    final state, all three observation kernels — against the oracle."""
    n, horizon, T = 517, 35, 90
    env = BatchedOvercookedEnv(name, n, horizon=horizon, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5,
                               seed=sum(map(ord, name)))
    rs = cpu.random_start(sum(map(ord, name)), 0.5, True)
    ref = np.zeros((n, env.state_words), np.int32)
    cpu.reset_random(env._tab_host, env._starts_host, ref, rs)
    assert np.array_equal(_np(env.state), ref)
    rng = np.random.RandomState(len(name))
    acts = _random_actions(rng, T, n, 0.4)
    want = cpu.rollout(env._tab_host, env._starts_host, ref, acts, horizon=horizon, flags=1, n_threads=2, rs=rs)
    got = env.rollout(torch.from_numpy(acts).cuda())
    for g, w in zip(got, want):
        assert np.array_equal(_np(g), w)
    assert np.array_equal(_np(env.state), ref)
    l = env.layouts[0]
    enc = env.lossless_state_encoding(dtype=torch.uint8)
    assert np.array_equal(_np(enc).astype(np.int32), cpu.encode_lossless(env._tab_host, ref, l.width, l.height, horizon))
    f = _np(env.featurize_state(2))
    assert np.array_equal(f.astype(np.float64), cpu.featurize(env._tab_host, lut_bytes([l]), ref, 2))
    pt, cst, gpow = L.build_potential_tables([l], 0.99)
    assert np.array_equal(_np(env.potential(0.99)), cpu.potential(env._tab_host, pt, cst, gpow, ref))


def test_packed_event_codes_cover_every_event_pattern():
    """OVC_F_OUT_PACKED: decoding the 5-bit event codes gives back exactly the int32 event masks on every
    fixture transition (all 25 event types, deliveries of several recipes) and on finished-env steps."""
    from overcooked_ai_b200 import wire

    seen = set()
    for path in TRACE_FILES:
        tr = Trace(path)
        s0, a, s1, sparse, shaped, events = tr.flat()
        env = _env_for_trace(tr, len(s0), 0)
        env.state.copy_(torch.from_numpy(s0))
        full = env.rollout(torch.from_numpy(a[None]).cuda())
        env.state.copy_(torch.from_numpy(s0))
        out = env.alloc_rollout_out(1, packed=True)
        env.rollout(torch.from_numpy(a[None].astype(np.uint8)).cuda(), out=out)
        ev, dn = wire.decode_event_codes(_np(out[3]))
        assert np.array_equal(ev, _np(full[3])) and np.array_equal(_np(out[0]), _np(full[0])) and np.array_equal(_np(out[1]), _np(full[1]))
        seen |= set(np.unique(_np(out[3]).astype(np.int32) & 31).tolist()) | set(np.unique((_np(out[3]).astype(np.int32) >> 5) & 31).tolist())
    assert len(seen) >= 24, sorted(seen)
    env = BatchedOvercookedEnv("cramped_room", 64, horizon=3, auto_reset=False)
    acts = torch.zeros((5, 64, 2), dtype=torch.uint8, device="cuda")
    out = env.alloc_rollout_out(5, packed=True)
    env.rollout(acts, out=out)
    ev, dn = wire.decode_event_codes(_np(out[3]))
    assert dn[2:].all() and not dn[:2].any() and (ev[3:] == L.EVF_STEPPED_DONE).all()


def test_two_ranks_mixed_batch_on_gpus():
    """SURVEY 8(e) on hardware: 2 NCCL ranks (one per GPU), a config-3-shaped mixed batch sharded with
    dist.shard_segments, each rank's shard against the oracle, the reduced counters against the whole batch.  Needs two
    visible GPUs (skips on a single GPU)."""
    import os
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    port = 29600 + os.getpid() % 2000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(root, "tests", "_dist_gpu_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, PYTHONPATH=root, OMP_NUM_THREADS="1"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "DIST_GPU_OK" in out.stdout


def test_long_rollouts_are_cut_into_launches():
    """The rollout kernel addresses its rows with 32-bit element indices, so ovc_rollout cuts a rollout of more than 2^32
    env-steps into consecutive launches.  The cut itself (pointer arithmetic per transfer format, pot clocks across the
    cut) is exercised at a small size through the library's test hook, in a child process (the hook is read once)."""
    import os
    import subprocess
    import sys

    root = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
    code = r"""
import numpy as np, torch
from oracle import cpu
from overcooked_ai_b200 import wire
from overcooked_ai_b200.batched import BatchedOvercookedEnv
names, n, T = ["cramped_room", "counter_circuit"], 777, 53
rng = np.random.RandomState(2)
acts = rng.randint(0, 6, size=(T, n, 2)).astype(np.int32); acts[rng.rand(T, n, 2) < 0.4] = 5
env = BatchedOvercookedEnv(names, n, horizon=25, auto_reset=True)
state = env.state.cpu().numpy().copy()
want = cpu.rollout(env._tab_host, env._starts_host, state, acts, horizon=25, flags=1, n_threads=2)
got = env.rollout(torch.from_numpy(acts).cuda())                      # int32 formats, 8 launches of <= 7 transitions
for g, w in zip(got, want):
    assert np.array_equal(g.cpu().numpy(), w)
assert np.array_equal(env.state.cpu().numpy(), state)
env.reset()
out = env.alloc_rollout_out(T, codes=True)                            # one-byte actions in, 2-byte code words out
env.rollout(torch.from_numpy(wire.pack_actions(acts)).cuda(), out=out)
dense = env.expand_codes(out[3].cpu(), events=True)
for k, w in zip(("sparse", "shaped", "done", "events"), want):
    assert np.array_equal(dense[k].numpy(), w), k
env.reset()
out = env.alloc_rollout_out(T, packed=True)                           # uint8 actions, packed outputs
env.rollout(torch.from_numpy(acts.astype(np.uint8)).cuda(), out=out)
assert np.array_equal(out[0].cpu().numpy(), want[0]) and np.array_equal(out[1].cpu().numpy(), want[1])
print("CUT_OK")
"""
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, PYTHONPATH=root, OVC_K5_MAX_LAUNCH_STEPS="7"))
    assert out.returncode == 0 and "CUT_OK" in out.stdout, out.stdout[-1000:] + out.stderr[-3000:]
