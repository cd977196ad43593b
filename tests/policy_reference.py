"""float64 restatements of the policy kernels K7 (ovc_encode_linear), K9 (ovc_wide_layers) and K8 (ovc_policy_tail) and of
the action draw (ovc_sample_actions), with operands on which the kernels' float32 accumulation is exact.

Exactness: an accumulation out = sum_k a_k w_k + b is computed exactly by ANY summation order in float32 (a tensor core
that truncates while aligning its addends included) when every term and the bias are integer multiples of one power of two
g and sum |terms| + |bias| < 2^22 g: every partial sum is then a multiple of g below 2^22 g.  On such operands a kernel's
output is the round-to-nearest-even of a known value at each documented rounding point, so it must equal the
restatement bit for bit.  ``Certificate`` checks the premise per accumulation; a test asserts it before it compares, so a
broken premise does not read as a kernel bug."""
import numpy as np
import torch

from ppo_reference import log_softmax_at

EXACT_BITS = 22
_NONE = 1 << 20  # valuation of 0: no power of two bounds it


def bf16(x):
    """Round to nearest even bfloat16, as float64 (through float32: exact wherever a certificate holds)."""
    f = np.ascontiguousarray(np.asarray(x, np.float64).astype(np.float32))
    return torch.from_numpy(f).to(torch.bfloat16).double().numpy()


def torch_bf16(t):
    """bf16 rounding of a torch tensor, kept in its dtype."""
    return t.float().to(torch.bfloat16).to(t.dtype)


def leaky(z, slope):
    return np.where(z > 0, z, z * slope)


def valuation(x):
    """2-adic valuation of each element: the largest e with x a multiple of 2^e (a large number for 0)."""
    x = np.asarray(x, np.float64)
    m, e = np.frexp(np.abs(x))
    mi = (m * 2.0 ** 53).astype(np.int64)
    low = mi & -mi
    v = e.astype(np.int64) - 53 + np.frexp(low.astype(np.float64))[1].astype(np.int64) - 1
    return np.where(x == 0, _NONE, v)


def significant_bits(x):
    """Significant bits of each element (0 for 0)."""
    x = np.asarray(x, np.float64)
    top = np.frexp(np.abs(x))[1].astype(np.int64)
    return np.where(x == 0, 0, top - valuation(x))


class Certificate(object):
    """out[r, c] = sum_k a[r, k] w[c, k] + b[c]: ``log2_g`` [r, c], a power of two dividing every term and the bias, and
    ``abs_sum`` [r, c] = sum_k |a[r, k] w[c, k]| + |b[c]|."""

    def __init__(self, a, w, b):
        a, w, b = (np.asarray(t, np.float64) for t in (a, w, b))
        va, vw, vb = valuation(a), valuation(w), valuation(b)[None, :]
        # first a bound from the smallest valuations of a's row and of w's column
        self.log2_g = np.minimum(np.minimum(va.min(1)[:, None] + vw.min(1)[None, :], _NONE), vb)
        self.abs_sum = np.abs(a) @ np.abs(w).T + np.abs(b)[None, :]
        rows = np.flatnonzero(~self.exact().all(1))
        nz = [np.flatnonzero(row) for row in w]
        if len(rows) and max(len(k) for k in nz) <= 32:  # sparse w: the smallest valuation over each column's own terms
            v = va[rows]
            g = np.stack([(v[:, k] + vw[c, k]).min(1) if len(k) else np.full(len(rows), _NONE) for c, k in enumerate(nz)], 1)
            self.log2_g[rows] = np.minimum(np.minimum(g, _NONE), vb)

    def exact(self):
        """[r, c]: the accumulation is exact in float32 in any order."""
        return (self.abs_sum == 0) | (self.abs_sum < np.ldexp(1.0, EXACT_BITS + np.minimum(self.log2_g, 1000)))

    def holds(self):
        return bool(self.exact().all())


def linear(a, w, b):
    """(a w^T + b in float64, its Certificate)."""
    a, w, b = (np.asarray(t, np.float64) for t in (a, w, b))
    return a @ w.T + b, Certificate(a, w, b)


def dyadic(rng, shape, max_int, exps, density=1.0, signed=True):
    """Integers in [-max_int, max_int] ([0, max_int] unsigned) times 2^-e with e drawn from ``exps``, each element zero with
    probability 1 - density."""
    k = rng.randint(-max_int if signed else 0, max_int + 1, size=shape)
    e = rng.choice(np.asarray(exps), size=shape)
    return np.ldexp(k.astype(np.float64), -e) * (rng.random_sample(shape) < density)


# ---------------------------------------------------------------------------------------------------------------- K7
def k7_reference(obs, wt, bias, slope):
    """ovc_encode_linear on the materialised observation: bf16(leaky(obs . W + b)).  obs [rows, W*H*26] (the oracle's
    lossless encoding, views flattened), wt [W*H*26, n_out] (the table: W transposed).  Returns (out, [Certificate])."""
    z, cert = linear(obs, np.asarray(wt, np.float64).T, bias)
    return bf16(leaky(z, slope)), [cert]


def k7_operands(rng, n_in, n_out):
    """A K7 table and bias: signed dyadic, 8 significant bits at most (exact in bfloat16)."""
    return dyadic(rng, (n_in, n_out), 7, range(7), density=0.3), dyadic(rng, n_out, 127, [6])


# ---------------------------------------------------------------------------------------------------------------- K9
def k9_reference(a0, w1, b1, w2, b2, slope):
    """ovc_wide_layers: a1 = bf16(leaky(a0 W1^T + b1)), z2 = bf16(a1 W2^T + b2).  Returns (z2, [Certificate] x 2, (z1, z2
    before rounding))."""
    z1, c1 = linear(a0, w1, b1)
    a1 = bf16(leaky(z1, slope))
    z2, c2 = linear(a1, w2, b2)
    return bf16(z2), [c1, c2], (z1, z2)


def k9_operands(rng, m):
    """a0 [m, 512], w1 [512, 512], b1, w2 [160, 512], b2: sparse signed dyadic weights; layer 1 sums need up to ~15
    significant bits (an 11-bit accumulator would lose them)."""
    w1 = dyadic(rng, (512, 512), 7, range(6), density=16 / 512)
    w2 = dyadic(rng, (160, 512), 3, [0, 1], density=8 / 512)
    return k9_rows(rng, m), w1, dyadic(rng, 512, 255, [7]), w2, dyadic(rng, 160, 255, [9])


def k9_rows(rng, m):
    return dyadic(rng, (m, 512), 15, [2], density=0.6)


# ---------------------------------------------------------------------------------------------------------------- K8
def k8_reference(x, w_first, b_first, w_hidden, b_hidden, w_heads, b_heads, in_slope, slope):
    """ovc_policy_tail's heads: bf16(leaky(x, in_slope)) on load, bf16(leaky(.)) after each 64-wide layer, heads in
    float32 (exact here).  Returns (heads [rows, 8], [Certificate] per layer)."""
    a = bf16(leaky(np.asarray(x, np.float64), in_slope))
    z, c = linear(a, w_first, b_first)
    certs = [c]
    a = bf16(leaky(z, slope))
    for l in range(len(w_hidden)):
        z, c = linear(a, w_hidden[l], b_hidden[l])
        certs.append(c)
        a = bf16(leaky(z, slope))
    s, c = linear(a, w_heads, b_heads)
    certs.append(c)
    return s, certs


def k8_operands(rng, n_rows, k0, n_hidden):
    """x [n_rows, k0] and the tail's weights: sparse signed dyadic (use ``certified_rows`` to re-draw the few rows whose
    chain of up to ten accumulations is not certified exact)."""
    w_first = dyadic(rng, (64, k0), 3, [1, 2], density=min(1.0, 8 / k0))
    b_first = dyadic(rng, 64, 15, [4])
    w_hidden = dyadic(rng, (n_hidden, 64, 64), 3, [1, 2], density=6 / 64)
    b_hidden = dyadic(rng, (n_hidden, 64), 15, [4])
    w_heads = dyadic(rng, (8, 64), 7, [2, 3], density=0.25)
    b_heads = dyadic(rng, 8, 15, [4])
    return k8_rows(rng, n_rows, k0), w_first, b_first, w_hidden, b_hidden, w_heads, b_heads


def k8_rows(rng, n, k0):
    return dyadic(rng, (n, k0), 15, [2, 3], density=0.5)


def certified_rows(rng, x, draw_rows, restate, tries=8):
    """Re-draw (``draw_rows(rng, n)``) the rows of x whose accumulations are not all certified exact by
    ``restate(x) -> (out, [Certificate])``; the rows of these kernels are independent.  Returns (x, out, certificates)."""
    for _ in range(tries):
        out, certs = restate(x)[:2]
        bad = np.zeros(len(x), bool)
        for c in certs:
            bad |= ~c.exact().all(1)
        if not bad.any():
            return x, out, certs
        x = x.copy()
        x[bad] = draw_rows(rng, int(bad.sum()))
    raise AssertionError("could not draw certified operands")


# ------------------------------------------------------------------------------------------------------------ the draw
def philox4x32_10(key, c):
    """numpy restatement of Philox4x32-10 (Salmon et al.): key uint64, c uint32[n, 4] -> uint32[n, 4]."""
    c = [c[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key & 0xFFFFFFFF), np.uint64(key >> 32)
    M = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return np.stack(c, 1).astype(np.uint32)


def gumbel_scores(scores, seed, step, n_actions=6, rows=None):
    """scores[:, i] - log(-log u_i) of the ovc_sample_actions definition: counter (row lo, row hi, step lo, 2 step hi + i / 4).
    ``rows``: the row id each score row is drawn on (the joint row of a row map); default 0, 1, ..."""
    rows = np.arange(len(scores), dtype=np.uint64) if rows is None else np.asarray(rows).astype(np.uint64)
    step = int(step)
    ctr = np.stack([rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32), np.full_like(rows, step & 0xFFFFFFFF),
                    np.full_like(rows, (step >> 32) << 1)], 1).astype(np.uint32)
    d = np.concatenate([philox4x32_10(seed, ctr), philox4x32_10(seed, ctr | np.array([0, 0, 0, 1], np.uint32))], 1)[:, :n_actions]
    u = ((d >> np.uint32(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    return np.asarray(scores)[:, :n_actions] - np.log(-np.log(u))


def check_draw(actions, scores, seed, step, n_actions=6, rows=None, row_sensitive=False):
    """actions == the ovc_sample_actions definition applied to ``scores`` at ``step``, row i drawn on row id ``rows[i]``
    (default i) (near-ties exempt).  ``row_sensitive``: also require that the definition at row ids rows + 1 draws another
    action on some clear row, so that scores whose spread leaves no room for the noise cannot hide a draw on the wrong
    row id."""
    if n_actions == 1:
        assert (actions == 0).all()
        return
    v = gumbel_scores(scores, seed, step, n_actions, rows)
    top2 = np.sort(v, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-4  # libm and the device logf differ in the last bits: near-ties may flip
    assert clear.mean() > 0.995 and np.array_equal(actions[clear], v.argmax(1)[clear])
    if row_sensitive:
        ids = (np.arange(len(scores)) if rows is None else np.asarray(rows, np.int64)) + 1
        other = gumbel_scores(scores, seed, step, n_actions, ids).argmax(1)
        assert (other[clear] != v.argmax(1)[clear]).any(), "the draw does not depend on the row id"
    assert actions.min() >= 0 and actions.max() < n_actions


def check_logp(logp, scores, actions, n_actions):
    want = log_softmax_at(scores, actions, n_actions)
    assert (np.abs(np.asarray(logp, np.float64) - want) <= 1e-5 * (1 + np.abs(want))).all(), np.abs(logp - want).max()


# ------------------------------------------------------------------------------------------------- exact network weights
HEAD_SHIFT = 6  # the heads are integers times 2^-6: logits spread over a few units


def plane_bounds(cook_time=20):
    """Largest value of each lossless_state_encoding plane: ingredient counts 3, cook time remaining the cook time, else 1."""
    b = np.ones(26)
    b[16:20] = 3
    b[20] = cook_time
    return b


def exact_cnn(width, height, seed, cook_time=20, caps=(15, 31, 63, 127, 255, 255, 255)):
    """An RllibShapedCNN with non-negative, sparse integer weights and biases (heads: integers times 2^-HEAD_SHIFT).  The
    largest value of every unit over ALL observations (interval bound from ``plane_bounds``) stays within its layer's cap
    (conv_initial, conv_0, conv_1, the dense layers, the heads in units of 2^-HEAD_SHIFT), so every activation and every
    pre-bias product is a non-negative integer of at most 8 bits: exact in bfloat16 and float32 in any summation order, and
    on the positive branch of every leaky ReLU.  The float64 network, its bf16-at-every-layer version, library bf16 GEMMs
    and K7 / K9 / K8 then all compute the same numbers.  The caps grow layer by layer so that every unit has several
    inputs."""
    from overcooked_ai_b200.selfplay import RllibShapedCNN

    rng = np.random.RandomState(seed)
    cnn = RllibShapedCNN(width, height).eval()

    def wire(w, b, bound_in, cap, draw):
        """Zeroes w [out, in...] and gives each output up to 6 inputs (index tuples from draw()) of weight 1..3 within cap."""
        w.zero_()
        out_bound = np.zeros(w.shape[0])
        for o in range(w.shape[0]):
            bias = int(rng.randint(0, 4))
            bound = bias
            for idx in draw(6):
                wv = int(rng.choice([1, 1, 2, 3]))
                if bound + wv * bound_in[idx[0]] <= cap and w[(o,) + idx] == 0:
                    w[(o,) + idx] = wv
                    bound += wv * bound_in[idx[0]]
            b[o] = bias
            out_bound[o] = bound
        return out_bound

    with torch.no_grad():
        bound = plane_bounds(cook_time)
        for conv, cap in zip((cnn.conv_initial, cnn.conv_0, cnn.conv_1), caps):
            ci, k = conv.weight.shape[1], conv.weight.shape[2]
            bound = wire(conv.weight, conv.bias, bound, cap,
                         lambda n, ci=ci, k=k: [(int(rng.randint(ci)), int(rng.randint(k)), int(rng.randint(k))) for _ in range(n)])
        bound = np.repeat(bound, (width - 2) * (height - 2))  # torch's flatten order (c, x, y)
        for d, cap in zip(cnn.dense, caps[3:]):
            n_in = d.weight.shape[1]
            bound = wire(d.weight, d.bias, bound, cap, lambda n, n_in=n_in: [(int(rng.randint(n_in)),) for _ in range(n)])
        for head in (cnn.logits, cnn.value):
            wire(head.weight, head.bias, bound, caps[-1], lambda n: [(int(rng.randint(64)),) for _ in range(n)])
            head.weight.mul_(2.0 ** -HEAD_SHIFT), head.bias.mul_(2.0 ** -HEAD_SHIFT)
    return cnn


def cnn_forward64(cnn, obs):
    """The float64 forward of ``cnn`` on observations [M, 2, W, H, 26] (any dtype) -> (logits [2M, 6], value [2M])."""
    import copy

    ref = copy.deepcopy(cnn).double().cpu()
    o = torch.as_tensor(np.asarray(obs), dtype=torch.float64)
    o = o.reshape(-1, *o.shape[-3:]).permute(0, 3, 1, 2)
    with torch.no_grad():
        l, v = ref(o)
    return l.numpy(), v.numpy()
