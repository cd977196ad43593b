"""The LSTM PPO model on the host: RllibLSTMShapedCNN.load_keras_weights gives the reference Keras model's function
(ppo_rllib.py:89-238, restated in numpy), forward_sequence's resets equal fresh runs from zero state, and the tables K11
takes (gate permutation, [W_ih | W_hh], one bias sum) are the torch LSTM."""
import numpy as np
import pytest
import torch

from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibLSTMShapedCNN, lstm_gate_permutation

W, H, C, NF, HID, CELL = 5, 4, 26, 25, 64, 256


def _keras_weights(rng):
    s = 0.1
    conv = [(rng.normal(size=(5, 5, C, NF)) * s, rng.normal(size=NF) * s), (rng.normal(size=(3, 3, NF, NF)) * s, rng.normal(size=NF) * s),
            (rng.normal(size=(3, 3, NF, NF)) * s, rng.normal(size=NF) * s)]
    flat = (W - 2) * (H - 2) * NF
    dense = [(rng.normal(size=(flat, HID)) * s, rng.normal(size=HID) * s)] + [(rng.normal(size=(HID, HID)) * s, rng.normal(size=HID) * s) for _ in range(2)]
    lstm = (rng.normal(size=(HID, 4 * CELL)) * s, rng.normal(size=(CELL, 4 * CELL)) * s, rng.normal(size=4 * CELL) * s)
    logits, value = (rng.normal(size=(CELL, 6)) * s, rng.normal(size=6) * s), (rng.normal(size=(CELL, 1)) * s, rng.normal(size=1) * s)
    f32 = lambda ws: tuple(a.astype(np.float32).astype(np.float64) for a in ws)  # load_keras_weights takes float32 weights
    return [f32(p) for p in conv], [f32(p) for p in dense], f32(lstm), f32(logits), f32(value)


def _keras_forward(obs, h, c, conv, dense, lstm, logits, value, dense_slope):
    """numpy restatement of the Keras model over a sequence obs [L, B, W, H, C] (TimeDistributed layers): Conv2D 5x5 'same',
    3x3 'same', 3x3 'valid' with tf.nn.leaky_relu (0.2), Flatten over (x, y, channel), Dense with leaky ReLU, LSTM (gate
    order i, f, c, o, one bias, sigmoid / tanh), heads on the LSTM output."""
    def conv2d(x, k, b, same):
        kh, kw = k.shape[:2]
        if same:
            x = np.pad(x, ((0, 0), (kh // 2, kh // 2), (kw // 2, kw // 2), (0, 0)))
        wo, ho = x.shape[1] - kh + 1, x.shape[2] - kw + 1
        out = np.zeros((x.shape[0], wo, ho, k.shape[3]))
        for i in range(kh):
            for j in range(kw):
                out += x[:, i:i + wo, j:j + ho, :] @ k[i, j]
        return out + b

    lrelu = lambda z, a: np.where(z > 0, z, a * z)
    sig = lambda z: 1 / (1 + np.exp(-z))
    L, B = obs.shape[:2]
    x = obs.reshape(L * B, W, H, C)
    x = lrelu(conv2d(x, *conv[0], True), 0.2)
    x = lrelu(conv2d(x, *conv[1], True), 0.2)
    x = lrelu(conv2d(x, *conv[2], False), 0.2).reshape(L * B, -1)
    for k, b in dense:
        x = lrelu(x @ k + b, dense_slope)
    x = x.reshape(L, B, -1)
    kern, rec, bias = lstm
    out = []
    for t in range(L):
        z = x[t] @ kern + h @ rec + bias
        i, f, g, o = (z[:, q * CELL:(q + 1) * CELL] for q in range(4))
        c = sig(f) * c + sig(i) * np.tanh(g)
        h = sig(o) * np.tanh(c)
        out.append(h)
    y = np.stack(out)
    return y @ logits[0] + logits[1], (y @ value[0] + value[1])[..., 0], h, c


@pytest.mark.parametrize("dense_slope", [0.2, 0.3])
def test_lstm_policy_loads_the_reference_keras_model_weights(dense_slope):
    rng = np.random.RandomState(5)
    weights = _keras_weights(rng)
    L, B = 4, 3
    obs = (rng.rand(L, B, W, H, C) < 0.1).astype(np.float64) * rng.randint(1, 4, size=(L, B, W, H, C))
    h0, c0 = rng.normal(size=(B, CELL)) * 0.5, rng.normal(size=(B, CELL)) * 0.5  # a non-zero start state
    want_l, want_v, want_h, want_c = _keras_forward(obs, h0, c0, *weights, dense_slope)
    m = RllibLSTMShapedCNN(W, H, dense_slope=dense_slope).double().eval()
    m.load_keras_weights(*weights)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    with torch.no_grad():
        l, v, (h, c) = m.forward_sequence(t(obs).permute(0, 1, 4, 2, 3), t(h0), t(c0))
    for got, want in ((l, want_l), (v, want_v), (h, want_h), (c, want_c)):
        assert np.allclose(got.numpy(), want, atol=1e-10, rtol=1e-10)


def test_forward_sequence_resets_equal_fresh_runs():
    torch.manual_seed(0)
    m = RllibLSTMShapedCNN(W, H).double().eval()
    L, B = 7, 4
    obs = (torch.rand(L, B, C, W, H, dtype=torch.float64) < 0.1).double() * 2
    h0, c0 = torch.randn(B, CELL, dtype=torch.float64), torch.randn(B, CELL, dtype=torch.float64)
    reset = torch.zeros(L, B, dtype=torch.uint8)
    reset[3, 0] = reset[5, 0] = reset[2, 2] = reset[0, 3] = 1
    with torch.no_grad():
        l, v, _ = m.forward_sequence(obs, h0, c0, reset)
        for b in range(B):
            starts = [0] + [t for t in range(L) if reset[t, b]]
            bounds = sorted(set(starts)) + [L]
            for s, e in zip(bounds[:-1], bounds[1:]):
                zero = torch.zeros(1, CELL, dtype=torch.float64)
                hs, cs = (zero, zero) if reset[s, b] else (h0[b:b + 1], c0[b:b + 1])
                ls, vs, _ = m.forward_sequence(obs[s:e, b:b + 1], hs, cs)
                assert torch.allclose(l[s:e, b:b + 1], ls, atol=1e-12) and torch.allclose(v[s:e, b:b + 1], vs, atol=1e-12)


def test_lstm_tables_are_the_torch_lstm():
    torch.manual_seed(1)
    m = RllibLSTMShapedCNN(W, H).eval()
    with torch.no_grad():
        m.lstm.bias_hh.normal_()  # a torch-trained cell has two biases: the table holds their sum
    d = DenseGridPolicy(m, W, H, pad_to=16).eval()
    w, b, wo, bo = d.lstm_tables()
    perm = lstm_gate_permutation(CELL)
    assert sorted(perm.tolist()) == list(range(4 * CELL))
    # row 64 j + 8 (4 half + gate) + n is gate `gate` of unit 16 j + 8 half + n
    j, half, gate, n = 5, 1, 2, 3
    assert perm[64 * j + 8 * (4 * half + gate) + n] == gate * CELL + 16 * j + 8 * half + n
    assert w.dtype == torch.bfloat16 and w.shape == (4 * CELL, HID + CELL) and b.dtype == torch.float32 and wo.shape == (8, CELL)
    x, h, c = torch.randn(9, HID).double(), torch.randn(9, CELL).double(), torch.randn(9, CELL).double()
    x, h = x.bfloat16().double(), h.bfloat16().double()
    # the folded cell in float64: gates in permuted order, then back to (i, f, g, o) blocks
    z = torch.cat([x, h], 1) @ w.double().t() + b.double()
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(4 * CELL)
    i, f, g, o = z[:, inv].split(CELL, 1)
    c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
    h2 = torch.sigmoid(o) * torch.tanh(c2)
    ref = m.lstm.double()
    ref.weight_ih.data, ref.weight_hh.data = ref.weight_ih.data.bfloat16().double(), ref.weight_hh.data.bfloat16().double()
    ref.bias_ih.data = (m.lstm.bias_ih.float() + m.lstm.bias_hh.float()).double()
    ref.bias_hh.data.zero_()
    with torch.no_grad():
        want_h, want_c = ref(x, (h, c))
    assert torch.allclose(h2, want_h, atol=1e-12) and torch.allclose(c2, want_c, atol=1e-12)
    assert torch.equal(wo[:6].float(), m.logits.weight.bfloat16().float()) and torch.equal(wo[6].float(), m.value.weight[0].bfloat16().float())
    assert torch.equal(bo[:7], torch.cat([m.logits.bias, m.value.bias]).float()) and (wo[7] == 0).all() and bo[7] == 0


def test_lstm_policy_library_path_matches_the_model():
    """DenseGridPolicy.hidden_from (the library path to K11's input) is the model's trunk; K8's tables stop there too."""
    torch.manual_seed(2)
    m = RllibLSTMShapedCNN(W, H).double().eval()
    d = DenseGridPolicy(m, W, H, pad_to=16).double().eval()
    obs = (torch.rand(5, W, H, C, dtype=torch.float64) < 0.1).double() * 3
    with torch.no_grad():
        assert torch.allclose(d.hidden_from(obs.reshape(5, -1), 0), m.trunk(obs.permute(0, 3, 1, 2)), atol=1e-10)
    assert len(d.hidden_tables()) == 4 and d.dense_slope == 0.2
    with pytest.raises(AssertionError):
        d.tail_tables()
