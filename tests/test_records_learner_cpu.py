"""The records learner without a GPU: K12 (ovc_encode_linear_wgrad) is declared, exported and loadable, malformed calls are
refused at M = 0 (nothing is launched), and the differentiable fold carries a PPO loss's gradient to every parameter of
RllibShapedCNN exactly as its conv2d forward does (float64)."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import (DenseGridPolicy, RllibLSTMShapedCNN, RllibShapedCNN, SampleBatch, folded_layers,
                                         records_forward)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 4096  # an aligned stand-in address: with M = 0 nothing is dereferenced


def test_wgrad_entry_point_is_declared_exported_and_loadable():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    assert "ovc_encode_linear_wgrad" in set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    assert "ovc_encode_linear_wgrad" in _native.EXPORTED_SYMBOLS
    lib = _native.lib()
    assert hasattr(lib, "ovc_encode_linear_wgrad")
    assert lib.ovc_abi_version() == 5


def _wgrad(lib, layouts=A, n_layouts=1, states=A, swap=0, seat=-1, dz=A, dwt=A, m=0, w=5, h=4, n_out=512):
    return lib.ovc_encode_linear_wgrad(layouts, n_layouts, states, swap, seat, dz, dwt, m, 16, w, h, 400, n_out, None)


def test_wgrad_accepts_well_formed_empty_calls_and_refuses_malformed_ones():
    lib = _native.lib()
    for seat, swap in ((-1, 0), (0, 0), (1, A), (0, A)):
        assert _wgrad(lib, seat=seat, swap=swap) == 0, lib.ovc_last_error()
    assert _wgrad(lib, w=13, h=7, n_out=64, n_layouts=8) == 0, lib.ovc_last_error()  # long_cook_time's grid at 8 layouts
    for kw in (dict(layouts=0), dict(states=0), dict(dz=0), dict(dwt=0)):
        assert _wgrad(lib, **kw) != 0 and b"null" in lib.ovc_last_error(), kw
    for kw in (dict(dz=A + 4), dict(dwt=A + 8), dict(states=A + 4), dict(swap=A + 2, seat=0)):
        assert _wgrad(lib, **kw) != 0 and b"aligned" in lib.ovc_last_error(), kw
    for n_out in (0, 32, 100, 520):
        assert _wgrad(lib, n_out=n_out) == _native_badarg() and b"n_out" in lib.ovc_last_error(), n_out
    assert _wgrad(lib, n_layouts=9) == _native_unsupported() and b"8 layouts" in lib.ovc_last_error()
    assert _wgrad(lib, w=16, h=16) == _native_unsupported() and b"shared memory" in lib.ovc_last_error()  # 256 cells
    assert _wgrad(lib, w=12, h=8) == _native_unsupported()  # 96 cells: one past K7's limit too
    assert _wgrad(lib, w=17, h=4) != 0 and b"grid" in lib.ovc_last_error()
    assert _wgrad(lib, seat=2) != 0 and b"seat" in lib.ovc_last_error()
    assert _wgrad(lib, m=-1) != 0


def _code(name):
    """An error code's value, read from the header."""
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    return int(re.search(r"#define\s+%s\s+\((-?\d+)\)" % name, hdr).group(1))


def _native_badarg():
    return _code("OVC_E_BADARG")


def _native_unsupported():
    return _code("OVC_E_UNSUPPORTED")


def _fold_forward64(cnn, obs, W, H, pad_to):
    """The folded network in float64: folded_layers' matrices, leaky ReLU 0.2 after the convolutions, the model's dense
    slope after the dense layers, the heads last.  obs [B, W*H*26] in [x][y][plane] order."""
    layers = folded_layers(cnn, W, H, pad_to=pad_to)
    x = obs
    for i, (w, b) in enumerate(layers[:-1]):
        x = F.leaky_relu(F.linear(x, w, b), 0.2 if i < 3 else cnn.dense_slope)
    hv = F.linear(x, *layers[-1])
    n = cnn.logits.out_features
    return hv[:, :n], hv[:, n]


def _ppo_loss(logits, values, actions, old_logp, adv, targets, clip=0.05):
    logp_all = F.log_softmax(logits, dim=-1)
    ratio = torch.exp(logp_all.gather(1, actions[:, None]).squeeze(1) - old_logp)
    policy = -torch.min(ratio * adv, ratio.clamp(1 - clip, 1 + clip) * adv).mean()
    entropy = -(logp_all.exp() * logp_all).sum(-1).mean()
    return policy + 1e-4 * F.mse_loss(values, targets) - 0.1 * entropy


@pytest.mark.parametrize("W,H,pad_to", [(5, 4, 16), (5, 4, 1), (9, 5, 16), (4, 3, 8)])
def test_fold_gradient_equals_the_conv_models_gradient_in_float64(W, H, pad_to):
    torch.manual_seed(W * 10 + H + pad_to)
    cnn = RllibShapedCNN(W, H).double()
    with torch.no_grad():  # larger weights than the default init, so that every leaky ReLU sees both signs
        for p in cnn.parameters():
            p.mul_(3.0)
    B = 48
    rng = np.random.RandomState(W + H)
    obs = torch.from_numpy((rng.random_sample((B, W, H, 26)) < 0.15) * rng.randint(1, 4, size=(B, W, H, 26))).double()
    actions = torch.from_numpy(rng.randint(0, 6, size=B))
    old_logp = torch.from_numpy(rng.normal(-1.8, 0.1, size=B))
    adv, targets = torch.from_numpy(rng.normal(size=B)), torch.from_numpy(rng.normal(size=B))

    logits, values = cnn(obs.permute(0, 3, 1, 2))
    want_loss = _ppo_loss(logits, values, actions, old_logp, adv, targets)
    want = torch.autograd.grad(want_loss, list(cnn.parameters()))

    logits_f, values_f = _fold_forward64(cnn, obs.reshape(B, -1), W, H, pad_to)
    got_loss = _ppo_loss(logits_f, values_f, actions, old_logp, adv, targets)
    got = torch.autograd.grad(got_loss, list(cnn.parameters()))

    assert torch.allclose(logits_f, logits, rtol=1e-12, atol=1e-12) and torch.allclose(values_f, values, rtol=1e-12, atol=1e-12)
    for (name, _), g, w in zip(cnn.named_parameters(), got, want):
        assert g.abs().max() > 0, name
        assert torch.allclose(g, w, rtol=1e-9, atol=1e-12 * float(w.abs().max())), (name, float((g - w).abs().max()))


def test_folded_layers_hold_dense_grid_policys_values():
    """The differentiable fold and the module the rollouts evaluate hold the same numbers, padding included."""
    torch.manual_seed(3)
    cnn = RllibShapedCNN(5, 4)
    dense = DenseGridPolicy(cnn, 5, 4, pad_to=16)
    mods = list(dense.conv_as_linear) + list(dense.dense) + [dense.heads]
    layers = folded_layers(cnn, 5, 4, pad_to=16)
    assert len(layers) == len(mods)
    for (w, b), mod in zip(layers, mods):
        assert w.requires_grad and torch.equal(w.detach(), mod.weight) and torch.equal(b.detach(), mod.bias)


def test_records_forward_refuses_the_lstm_model():
    env = type("E", (), {})()
    with pytest.raises(AssertionError, match="forward_sequence"):
        records_forward(RllibLSTMShapedCNN(5, 4), env, None)
    batch = SampleBatch.__new__(SampleBatch)
    batch.env, batch.one_view = env, False
    batch.states = torch.zeros((1, 1, 16), dtype=torch.int32)
    with pytest.raises(AssertionError, match="forward_sequence"):
        batch.forward(RllibLSTMShapedCNN(5, 4), torch.zeros(1, dtype=torch.int64))
