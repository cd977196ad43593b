"""The PPO learner on the sample batch's records: K12 (ovc_encode_linear_wgrad) bit for bit against float64 enc^T dz on
operands whose float32 sums are exact in any order (``policy_reference.Certificate``), K12's bookkeeping, and
SampleBatch.forward against the float64 CNN, the conv model and path (b) (K2 bf16 + the folded GEMMs)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import policy_reference as P
from helpers import TRACE_FILES, TRACE_IDS, Trace
from oracle import cpu
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.selfplay import AgentPairRollout, RllibShapedCNN, SelfPlayRollout

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 12345.0


def _np(t):
    return t.cpu().numpy()


def _fits(l):
    return l.width * l.height * 19 * 64 * 2 + 4096 <= 227 * 1024


def _enc_rows(env, states, seat=None, swap=None):
    """The oracle's encoding of K12's rows: [rows, W*H*26] float64."""
    l = env.layouts[0]
    obs = cpu.encode_lossless(env._tab_host, states, l.width, l.height, env.horizon).astype(np.float64)
    if seat is None:
        return obs.reshape(2 * len(states), -1)
    p = seat ^ (np.zeros(len(states), np.int64) if swap is None else (swap != 0).astype(np.int64))
    return obs[np.arange(len(states)), p].reshape(len(states), -1)


def _wgrad_check(env, states, rng, n_out, seat=None, swap=None, max_int=3):
    """K12 on ``states`` (int32 [M, S] numpy) against enc^T dz in float64: dz rows past M hold NaN, dwt is pre-loaded and
    followed by sentinel rows."""
    enc = _enc_rows(env, states, seat, swap)
    rows = enc.shape[0]
    dz = P.dyadic(rng, (rows, n_out), max_int, [3])
    pre = P.dyadic(rng, (enc.shape[1], n_out), 8, [3])
    cert = P.Certificate(enc.T, dz.T, np.zeros(n_out))
    assert ((cert.abs_sum + np.abs(pre)) < np.ldexp(1.0, P.EXACT_BITS + np.minimum(cert.log2_g, -3))).all(), \
        "premise: the sums are not exact in float32"
    want = enc.T @ dz + pre
    dz_full = torch.full((rows + GUARD, n_out), float("nan"), dtype=torch.float32, device="cuda")
    dz_full[:rows] = torch.from_numpy(dz).float()
    dwt_full = torch.full((enc.shape[1] + GUARD, n_out), SENTINEL, dtype=torch.float32, device="cuda")
    dwt_full[:enc.shape[1]] = torch.from_numpy(pre).float()
    dwt = dwt_full[:enc.shape[1]]
    sw = None if swap is None else torch.from_numpy(swap.astype(np.int32)).cuda()
    env.encoded_linear_wgrad(torch.from_numpy(states).cuda(), dz_full, dwt, seat=seat, swap=sw)
    got = _np(dwt).astype(np.float64)
    assert np.array_equal(got, want), (n_out, seat, np.abs(got - want).max(), (got != want).sum())
    assert bool((dwt_full[enc.shape[1]:] == SENTINEL).all()), "K12 wrote past dwt"
    return enc


def _played(layout, n, horizon=60, seed=0, steps=25):
    env = BatchedOvercookedEnv(layout, n, horizon=horizon, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.6, seed=seed)
    rng = np.random.RandomState(seed)
    acts = rng.randint(0, 6, size=(steps, n, 2)).astype(np.int32)
    acts[rng.rand(steps, n, 2) < 0.4] = 5
    env.rollout(torch.from_numpy(acts).cuda())
    return env


# ---------------------------------------------------------------------------------------------------------------- K12
@pytest.mark.parametrize("path", TRACE_FILES, ids=TRACE_IDS)
def test_k12_exact_on_fixture_states(path):
    tr = Trace(path)
    if not _fits(tr.layout):
        pytest.skip("the table of this grid does not fit shared memory (K7 and K12 refuse it)")
    st = np.ascontiguousarray(tr.data["obs_states"])
    env = BatchedOvercookedEnv(tr.layout, 1, horizon=400)
    rng = np.random.RandomState(len(st))
    for n_out in (64, 512):
        _wgrad_check(env, st, rng, n_out)
    _wgrad_check(env, st, rng, 128, seat=0, swap=(rng.rand(len(st)) < 0.5).astype(np.int32))


@pytest.mark.parametrize("layout,n", [("cramped_room", 2 * 333 + 1), ("counter_circuit", 1027), ("long_cook_time", 777)])
def test_k12_exact_on_random_play(layout, n):
    """Random starts then random play (held objects, cooking pots, counter_circuit's > 32 object slots, long_cook_time's 13x7
    grid at the shared-memory limit); every n_out from one column slice to many; one view with mixed swap, both seats;
    the urgency plane exactly at its edge."""
    horizon = 60
    env = _played(layout, n, horizon, seed=n)
    assert _fits(env.layouts[0])
    st = _np(env.state)
    rng = np.random.RandomState(n)
    for n_out in (64, 128, 192, 256, 512, 1024):
        _wgrad_check(env, st, rng, n_out)
    swap = (rng.rand(n) < 0.5).astype(np.int32)
    for seat in (0, 1):
        _wgrad_check(env, st, rng, 256, seat=seat, swap=swap)
    _wgrad_check(env, st, rng, 64, seat=1)
    for t in (horizon - 40, horizon - 39):
        s = st.copy()
        s[:, 0] = t
        urgency = _wgrad_check(env, s, rng, 128).reshape(2 * n, -1, 26)[..., 25]
        assert (urgency == 1).all() if t == horizon - 39 else not urgency.any()


def test_k12_exact_on_several_layouts_per_call():
    from overcooked_ai_b200 import layout as L

    def compiles(name):
        try:
            L.compile_layout(name)
            return True
        except Exception:
            return False

    names = [n for n in L.layout_names() if compiles(n) and (L.compile_layout(n).width, L.compile_layout(n).height) == (5, 4)]
    assert len(names) >= 9
    rng = np.random.RandomState(9)
    for k, n in ((1, 1), (2, 67), (8, 8 * 129 + 3)):
        env = BatchedOvercookedEnv(names[:k], n, horizon=50, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=k)
        env.rollout(torch.from_numpy(rng.randint(0, 6, size=(12, n, 2)).astype(np.int32)).cuda())
        assert len(np.unique(env.env_layout_host)) == min(k, n)
        _wgrad_check(env, _np(env.state), rng, 192)
        _wgrad_check(env, _np(env.state), rng, 128, seat=0, swap=(rng.rand(n) < 0.5).astype(np.int32))
    env = BatchedOvercookedEnv(names[:9], 90, horizon=50)
    with pytest.raises(RuntimeError, match="more than 8 layouts"):
        env.encoded_linear_wgrad(env.state, torch.zeros((180, 64), device="cuda"), torch.zeros((520, 64), device="cuda"))


@pytest.mark.parametrize("m", [1, 31, 32, 33, 20000])
def test_k12_exact_at_tile_edges_and_large(m):
    """M = 1, a CTA's 32 warps' worth of records +- 1, and a large batch (many records per warp, every CTA busy)."""
    env = _played("cramped_room", m, seed=m + 1)
    rng = np.random.RandomState(m)
    st = _np(env.state)
    _wgrad_check(env, st, rng, 512, max_int=1 if m > 1000 else 3)
    _wgrad_check(env, st, rng, 64, seat=1, swap=(rng.rand(m) < 0.5).astype(np.int32), max_int=1 if m > 1000 else 3)


def test_k12_with_zero_records_leaves_dwt_alone():
    env = BatchedOvercookedEnv("cramped_room", 4, horizon=400)
    dwt = torch.full((520, 64), 3.0, device="cuda")
    env.encoded_linear_wgrad(env.state[:0], torch.zeros((1, 64), device="cuda")[:0], dwt)
    assert bool((dwt == 3.0).all())


# ---------------------------------------------------------------------------------------------------- SampleBatch.forward
def _check_forward_exact(batch, env, model, n_rows):
    idx = torch.randperm(n_rows, device="cuda")[: min(n_rows, 3000)]
    logits, values = batch.forward(model, idx)
    obs = _np(batch.observations(idx))
    if batch.one_view:
        obs = obs[:, None]
    want_l, want_v = P.cnn_forward64(model, obs)
    assert np.array_equal(_np(logits.detach()).astype(np.float64), want_l)
    assert np.array_equal(_np(values.detach()).astype(np.float64), want_v)
    assert len(np.unique(want_l)) > 8


def test_forward_on_exact_weights_is_the_float64_cnn():
    """Self-play, a self-play mixture and a one-view pair batch: forward() == cnn_forward64 on the oracle-checked encoding."""
    n, T = 256, 10
    model = P.exact_cnn(5, 4, seed=21).cuda()
    env = BatchedOvercookedEnv("cramped_room", n, horizon=7, auto_reset=True)
    b = SelfPlayRollout(env, model=model, seed=1).collect(T, 0.99, 0.95)
    _check_forward_exact(b, env, model, T * n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=7, auto_reset=True)
    partner = P.exact_cnn(5, 4, seed=22).cuda()
    b = SelfPlayRollout(env, model=model, partner=partner, bc_factor=0.5, seed=2).collect(T, 0.99, 0.95)
    assert b.partner_seat is not None and (_np(b.partner_seat) >= 0).any() and (_np(b.partner_seat) < 0).any()
    _check_forward_exact(b, env, model, T * n)
    env = BatchedOvercookedEnv("cramped_room", n, horizon=7, auto_reset=True)
    b = AgentPairRollout(env, (model, partner), random_seats=True, seed=3).collect(T, 0.99, 0.95)
    assert b.one_view and len(np.unique(_np(b.partner_seat))) == 2
    _check_forward_exact(b, env, model, T * n)


def _random_batch(one_view=False, layout="cramped_room", n=512, T=8, seed=0):
    torch.manual_seed(seed)
    env = BatchedOvercookedEnv(layout, n, horizon=400, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=seed)
    W, H = env.layouts[0].width, env.layouts[0].height
    model = RllibShapedCNN(W, H).cuda()
    if one_view:
        b = AgentPairRollout(env, (model, copy.deepcopy(model)), random_seats=True, seed=seed).collect(T, 0.99, 0.95)
    else:
        b = SelfPlayRollout(env, model=model, seed=seed).collect(T, 0.99, 0.95, keep_logits=True)
    return env, model, b, T * n


@pytest.mark.parametrize("one_view", [False, True], ids=["two_views", "one_view"])
def test_forward_on_random_weights_is_the_conv_model_within_bf16(one_view):
    env, model, b, n_rows = _random_batch(one_view)
    idx = torch.arange(n_rows, device="cuda")
    logits, values = b.forward(model, idx)
    obs = b.observations(idx)
    obs = obs.view(-1, *obs.shape[-3:]).permute(0, 3, 1, 2)
    with torch.no_grad():
        want_l, want_v = model(obs)
    scale = float(want_l.abs().max())
    assert (logits.detach() - want_l).abs().max() <= 0.03 * scale + 1e-3
    assert (values.detach() - want_v).abs().max() <= 0.03 * float(want_v.abs().max()) + 1e-3
    assert torch.equal(logits.detach(), b.forward(model, idx, fused_first_layer=True)[0].detach())
    if not one_view:  # the behaviour policy's logp is close to the learner's: the mismatch the example prints
        lp = F.log_softmax(logits.detach(), -1).gather(1, b.actions.view(-1, 1).long()).squeeze(1)
        assert (lp - b.logp.view(-1)).abs().max() < 0.05


def _example_loss(logits, values, b, rows, adv, clip=0.05):
    logp_all = F.log_softmax(logits, dim=-1)
    logp = logp_all.gather(1, b.actions.view(-1)[rows, None].long()).squeeze(1)
    ratio = torch.exp(logp - b.logp.view(-1)[rows])
    a = adv[rows]
    policy = -torch.min(ratio * a, ratio.clamp(1 - clip, 1 + clip) * a).mean()
    entropy = -(logp_all.exp() * logp_all).sum(-1).mean()
    return policy + 1e-4 * F.mse_loss(values, b.value_targets.view(-1)[rows]) - 0.1 * entropy


def _reference_forward(model, b, idx):
    """records_forward with K7 / K12 replaced by float32 library math on K2's float32 observation: the first layer's sums
    in float32 (a GEMM with float32 accumulation and no TF32), its output rounded to bf16 once after the leaky ReLU, as K7
    rounds it; autograd gives its weight gradient as a float32 GEMM.  Every other layer is records_forward's."""
    from overcooked_ai_b200.selfplay import folded_layers

    assert not torch.backends.cuda.matmul.allow_tf32
    layers = folded_layers(model, 5, 4, pad_to=16)
    bf = lambda t: t.to(torch.bfloat16)
    obs = b.observations(idx)
    w0, b0 = layers[0]
    x = F.leaky_relu(F.linear(obs.reshape(-1, w0.shape[1]), bf(w0).float(), bf(b0).float()), 0.2).to(torch.bfloat16)
    for i, (w, bb) in enumerate(layers[1:-1], 1):
        x = F.leaky_relu(F.linear(x, bf(w), bf(bb)), 0.2 if i < 3 else model.dense_slope)
    wh, bh = layers[-1]
    hv = F.linear(x.float(), bf(wh).float(), bf(bh).float())
    return hv[:, :6], hv[:, 6]


@pytest.mark.parametrize("one_view", [False, True], ids=["two_views", "one_view"])
def test_forward_gradients(one_view):
    """The example's loss on one minibatch through forward() (K7 / K12) against the same network with a float32 first
    layer: every parameter gradient agrees to float32 summation order (plus the rare bf16 rounding flip a different
    summation order causes in the first layer's output).  Path (b) (K2's bf16 observation, bf16 GEMMs, whose first-layer
    weight gradient is rounded to bf16) agrees to bf16 accuracy."""
    env, model, b, n_rows = _random_batch(one_view, seed=5)
    idx = torch.randperm(n_rows, device="cuda")[:2048]
    rows = idx if one_view else (2 * idx[:, None] + torch.arange(2, device="cuda")).view(-1)
    adv = b.advantages.view(-1)
    adv = (adv - adv.mean()) / (adv.std() + 1e-8)
    grads = {}
    for k, fwd in (("records", lambda: b.forward(model, idx)), ("f32_first_layer", lambda: _reference_forward(model, b, idx)),
                   ("b", lambda: b.forward(model, idx, fused_first_layer=False))):
        model.zero_grad(set_to_none=True)
        _example_loss(*fwd(), b, rows, adv).backward()
        grads[k] = [p.grad.detach().clone() for p in model.parameters()]
    for (name, _), g, w, g_b in zip(model.named_parameters(), grads["records"], grads["f32_first_layer"], grads["b"]):
        err = float((g - w).norm() / (w.norm() + 1e-30))
        assert err < 5e-3, (name, err)
        err_b = float((g_b - w).norm() / (w.norm() + 1e-30))
        assert err_b < 0.1, (name, err_b)


def test_first_layer_backward_is_obs_transposed_times_dz():
    """The first layer's weight gradient alone: K12 against the float32 GEMM obs^T dz on K2's observation."""
    env, model, b, n_rows = _random_batch(False, seed=7)
    from overcooked_ai_b200.selfplay import _RecordsFirstLayer, folded_layers

    idx = torch.arange(n_rows, device="cuda")
    recs = b.states.view(-1, b.states.shape[-1]).index_select(0, idx)
    w0, b0 = [t.detach().clone().requires_grad_(True) for t in folded_layers(model, 5, 4)[0]]
    y = _RecordsFirstLayer.apply(w0, b0, env, recs, None, None)
    g = torch.randn(y.shape, device="cuda").to(torch.bfloat16)
    y.backward(g)
    dz = g.float() * torch.where(y.detach() > 0, 1.0, 0.2)
    obs = b.observations(idx).view(y.shape[0], -1).double()
    want_w = (dz.double().t() @ obs).float()
    assert torch.allclose(w0.grad, want_w, rtol=1e-4, atol=1e-4 * float(want_w.abs().max()))
    assert torch.allclose(b0.grad, dz.sum(0), rtol=1e-4, atol=1e-3)
