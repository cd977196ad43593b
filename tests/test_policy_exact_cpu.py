"""The exact-operand references of tests/policy_reference.py on the host: their premises hold, the K7 / K9 / K8
restatements composed on DenseGridPolicy's kernel tables are the network, and the exact-weight network computes the same
numbers in float64, folded, and with bfloat16 rounding after every layer."""
import numpy as np
import torch
import torch.nn.functional as F

import policy_reference as P
from overcooked_ai_b200.selfplay import DenseGridPolicy


def test_valuation_and_certificate():
    x = np.array([0.0, 1.0, 3.0, 0.75, -0.375, 2.0 ** -30, 6.0 * 2 ** 40])
    assert P.valuation(x)[1:].tolist() == [0, 0, -2, -3, -30, 41]
    assert P.significant_bits(x).tolist() == [0, 1, 2, 2, 2, 1, 2]
    a, w, b = np.array([[2.0 ** 21, 1.0]]), np.array([[1.0, 1.0]]), np.array([0.5])
    assert not P.Certificate(a, w, b).holds()  # 2^21 + 1.5 > 2^22 * 0.5
    assert P.Certificate(a, w, np.array([1.0])).holds()
    assert P.Certificate(np.array([[1.0, 2.0 ** -20]]), np.array([[1.0, 0.0]]), np.array([0.0])).holds()  # the 0 weight's term is 0


def test_builders_certificates_hold_and_need_more_than_11_bits():
    rng = np.random.RandomState(0)
    a0, w1, b1, w2, b2 = P.k9_operands(rng, 300)
    for slope in (0.0, 0.25, 1.0):
        a0, z2, certs = P.certified_rows(rng, a0, P.k9_rows, lambda x: P.k9_reference(x, w1, b1, w2, b2, slope))
        assert all(c.holds() for c in certs)
        z1, z2_exact = P.k9_reference(a0, w1, b1, w2, b2, slope)[2]
        assert (P.significant_bits(z1) > 11).mean() > 0.05 and (P.significant_bits(z2_exact) > 11).mean() > 0.3
        assert np.array_equal(P.bf16(z2), z2) and not np.array_equal(z2, z2_exact)
    ops = P.k8_operands(rng, 500, 96, 8)
    x, heads, certs = P.certified_rows(rng, ops[0], lambda r, n: P.k8_rows(r, n, 96), lambda x: P.k8_reference(x, *ops[1:], 0.25, 0.5))
    assert len(certs) == 10 and all(c.holds() for c in certs) and (P.significant_bits(heads) > 11).mean() > 0.3
    wt, b = P.k7_operands(rng, 520, 128)
    obs = rng.randint(0, 4, size=(40, 520)) * (rng.rand(40, 520) < 0.05)
    out, certs = P.k7_reference(obs, wt, b, 0.5)
    assert certs[0].holds() and np.array_equal(P.bf16(wt), wt)


def _tables64(d):
    wt0, b0 = d.first_layer_table()
    f = lambda ts: [t.double().numpy() for t in ts]
    return f((wt0, b0)), f(d.wide_tables()), f(d.tail_tables())


def test_restatements_on_the_kernel_tables_are_the_dense_policy():
    """K7 -> K9 -> K8 restated on the tables DenseGridPolicy hands the kernels equal the dense policy's own float64
    forward with bf16 rounding after every layer: the restatements are the network (exact weights: every number is exact)."""
    cnn = P.exact_cnn(5, 4, seed=1)
    d = DenseGridPolicy(cnn, 5, 4, pad_to=16).to(torch.bfloat16).eval()
    (wt0, b0), (w1, b1, w2, b2), (wf, bf, wh, bh, wo, bo) = _tables64(d)
    rng = np.random.RandomState(1)
    obs = (rng.randint(0, 3, size=(64, 520)) * (rng.rand(64, 520) < 0.08)).astype(np.float64)
    a0, c7 = P.k7_reference(obs, wt0, b0, 0.2)
    z2, c9, _ = P.k9_reference(a0, w1, b1, w2, b2, 0.2)
    heads, c8 = P.k8_reference(z2, wf, bf, wh, bh, wo, bo, 0.2, 0.3)
    assert all(c.holds() for c in c7 + c9 + c8)
    d64 = DenseGridPolicy(cnn.double(), 5, 4, pad_to=16).double().eval()
    with torch.no_grad():
        x = torch.from_numpy(obs)
        for lin in d64.conv_as_linear:
            x = P.torch_bf16(F.leaky_relu(lin(x), 0.2))
        for lin in d64.dense:
            x = P.torch_bf16(F.leaky_relu(lin(x), 0.3))
        want = d64.heads(x).numpy()
    assert np.array_equal(heads[:, :7], want[:, :7]) and len(np.unique(heads[:, :6])) > 10


def test_exact_weight_network_is_exact_in_every_form():
    """The exact-weight RllibShapedCNN: float64 CNN == float64 DenseGridPolicy == both with bf16 rounding after every layer,
    on observations at the planes' largest values; every unit stays within its bound."""
    for W, H, seed in ((5, 4, 2), (5, 5, 3), (9, 5, 4)):
        cnn = P.exact_cnn(W, H, seed=seed)
        assert all((p >= 0).all() for p in cnn.parameters())
        rng = np.random.RandomState(seed)
        bound = P.plane_bounds()
        obs = np.floor(rng.rand(40, 2, W, H, 26) * (bound + 1)) * (rng.rand(40, 2, W, H, 26) < 0.3)
        obs[0] = bound  # every plane at its largest value
        logits, value = P.cnn_forward64(cnn, obs)
        c64 = P.exact_cnn(W, H, seed=seed).double()
        x = torch.from_numpy(obs.reshape(-1, W, H, 26)).permute(0, 3, 1, 2)
        with torch.no_grad():
            for conv in (c64.conv_initial, c64.conv_0, c64.conv_1):
                x = P.torch_bf16(F.leaky_relu(conv(x), 0.2))
                assert x.max() <= 255
            x = x.flatten(1)
            for lin in c64.dense:
                x = P.torch_bf16(F.leaky_relu(lin(x), 0.3))
                assert x.max() <= 255
            l_bf, v_bf = c64.logits(x), c64.value(x).squeeze(-1)
            d64 = DenseGridPolicy(c64, W, H, pad_to=16).double().eval()
            l_d, v_d = d64(torch.from_numpy(obs.reshape(80, -1)))
        for got in ((l_bf, v_bf), (l_d, v_d)):
            assert np.array_equal(got[0].numpy(), logits) and np.array_equal(got[1].numpy(), value)
        assert np.array_equal(P.bf16(logits), logits) and logits.max() <= 4 and len(np.unique(logits)) > 8, np.unique(logits)
