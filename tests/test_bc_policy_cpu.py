"""BCPolicy (the PPO_BC partner) on the CPU: the reference's Keras weights load into the function the Keras model computes,
and tables() hands K10 the same weights with the heads padded to 8."""
import numpy as np
import torch

from overcooked_ai_b200.selfplay import BCPolicy


def keras_bc(x, dense, logits):
    """numpy restatement of behavior_cloning_tf2's MLP: Dense ReLU layers with kernels (in, out), then the logits."""
    for k, b in dense:
        x = np.maximum(x @ k + b, 0.0)
    return x @ logits[0] + logits[1]


def _weights(rng, n_hidden_layers, n_actions):
    """Keras kernels and biases, float32 values (what the model stores) held in float64."""
    f32 = lambda a: a.astype(np.float32).astype(np.float64)
    dims = [96] + [64] * n_hidden_layers
    dense = [(f32(rng.normal(size=(dims[i], dims[i + 1])) / 8), f32(rng.normal(size=dims[i + 1]))) for i in range(n_hidden_layers)]
    return dense, (f32(rng.normal(size=(64, n_actions))), f32(rng.normal(size=n_actions)))


def test_load_keras_weights_computes_the_keras_model():
    rng = np.random.RandomState(0)
    for n_layers, n_actions in ((1, 6), (2, 6), (3, 4)):
        dense, logits = _weights(rng, n_layers, n_actions)
        bc = BCPolicy(num_hidden_layers=n_layers, num_actions=n_actions).double().load_keras_weights(dense, logits)
        x = rng.randint(-8, 20, size=(50, 96)).astype(np.float64)
        with torch.no_grad():
            got = bc(torch.from_numpy(x)).numpy()
        assert np.allclose(got, keras_bc(x, dense, logits), rtol=1e-12, atol=1e-9)


def test_tables_are_the_weights_in_bf16_with_padded_heads():
    rng = np.random.RandomState(1)
    for n_layers, n_actions in ((1, 6), (2, 6), (3, 7)):
        dense, logits = _weights(rng, n_layers, n_actions)
        bc = BCPolicy(num_hidden_layers=n_layers, num_actions=n_actions).load_keras_weights(dense, logits)
        w1, b1, wh, bh, wo, bo = bc.tables()
        bf = lambda a: torch.as_tensor(a, dtype=torch.float32).to(torch.bfloat16)
        assert [t.dtype for t in (w1, b1, wh, bh, wo, bo)] == [torch.bfloat16, torch.float32] * 3
        assert tuple(w1.shape) == (64, 96) and tuple(wh.shape) == (n_layers - 1, 64, 64) and tuple(bh.shape) == (n_layers - 1, 64)
        assert tuple(wo.shape) == (8, 64) and tuple(bo.shape) == (8,)
        assert all(t.is_contiguous() for t in (w1, b1, wh, bh, wo, bo))
        assert torch.equal(w1, bf(dense[0][0].T)) and torch.equal(b1, torch.as_tensor(dense[0][1], dtype=torch.float32))
        for l in range(n_layers - 1):
            assert torch.equal(wh[l], bf(dense[l + 1][0].T)) and torch.equal(bh[l], torch.as_tensor(dense[l + 1][1], dtype=torch.float32))
        assert torch.equal(wo[:n_actions], bf(logits[0].T)) and torch.equal(bo[:n_actions], torch.as_tensor(logits[1], dtype=torch.float32))
        assert not wo[n_actions:].any() and not bo[n_actions:].any()  # padding, and a zero value row
