"""Behaviour-cloning training on the H100 (ovc_bc_train_epoch, include/ovc_bc.h): epochs against a float64 restatement of the
header's step, independence of the models of one launch, and the reference's own greedy games end to end."""
import math

import numpy as np
import pytest
import torch

from helpers import GOLD
from overcooked_ai_b200 import _bc_native, bc as B
from overcooked_ai_b200.batched import BatchedOvercookedEnv
from overcooked_ai_b200.greedy import GreedyHumanModel
from overcooked_ai_b200.selfplay import AgentPairRollout

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24  # float32's unit roundoff


def _golden_dataset():
    d = np.load(GOLD + "/greedy_cramped_room.npz")
    env = BatchedOvercookedEnv("cramped_room", 1, horizon=400)
    X, Y = B.bc_dataset(env, d["states"].reshape(-1, 16), d["actions"].reshape(-1, 2))
    return d, X, Y


# --- the float restatement of include/ovc_bc.h's epoch -------------------------------------------------------------------

def _layers(flat, L, A):
    out, o = [], 0
    for n_out, n_in in B.layer_shapes(L, A):
        out.append((flat[o:o + n_out * n_in].view(n_out, n_in), flat[o + n_out * n_in:o + n_out * n_in + n_out]))
        o += n_out * n_in + n_out
    return out


def _forward(lay, x):
    acts = [x]
    for W, b in lay[:-1]:
        acts.append(torch.relu(acts[-1] @ W.T + b))
    W, b = lay[-1]
    return acts, acts[-1] @ W.T + b


def ref_epoch(p, m, v, t, X, Y, train, val, batch, L, A, lr, dt):
    """One epoch in dtype dt on the CPU, in the header's order.  Returns (p, m, v, t, stats [4], logits of every row in
    the order they were taken, training rows first)."""
    p, m, v = p.to(dt).clone(), m.to(dt).clone(), v.to(dt).clone()
    c1, c2 = torch.tensor(0.1, dtype=torch.float32).to(dt), torch.tensor(0.001, dtype=torch.float32).to(dt)
    stats, logits = [0.0, 0, 0.0, 0], []
    for r0 in range(0, len(train), batch):
        idx = torch.from_numpy(train[r0:r0 + batch])
        n, x, y = len(idx), X[idx].to(dt), Y[idx]
        lay = _layers(p, L, A)
        acts, z = _forward(lay, x)
        loss = torch.logsumexp(z, 1) - z[torch.arange(n), y]
        stats[0] += float(loss.double().sum())
        stats[1] += int((z.argmax(1) == y).sum())
        logits.append(z.double())
        d = (torch.softmax(z, 1) - torch.nn.functional.one_hot(y, A).to(dt)) / n
        grads = [None] * (L + 1)
        for l in range(L, -1, -1):
            W = lay[l][0]
            grads[l] = torch.cat([(d.T @ acts[l]).reshape(-1), d.sum(0)])
            if l > 0:
                d = (d @ W) * (acts[l] > 0).to(dt)
        g = torch.cat(grads)
        t += 1
        alpha = torch.tensor(lr * math.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t), dtype=torch.float32).to(dt)
        m = m + (g - m) * c1
        v = v + (g * g - v) * c2
        p = p - alpha * m / (torch.sqrt(v) + torch.tensor(1e-7, dtype=torch.float32).to(dt))
    lay = _layers(p, L, A)
    for r0 in range(0, len(val), batch):
        idx = torch.from_numpy(val[r0:r0 + batch])
        _, z = _forward(lay, X[idx].to(dt))
        y = Y[idx]
        stats[2] += float((torch.logsumexp(z, 1) - z[torch.arange(len(idx)), y]).double().sum())
        stats[3] += int((z.argmax(1) == y).sum())
        logits.append(z.double())
    return p, m, v, t, stats, torch.cat(logits) if logits else torch.zeros((0, A), dtype=torch.float64)


# --- the library call, every output inside sentinels -----------------------------------------------------------------

PAD = 64
SENTINEL = -7777.0


class Buffers(object):
    """params / adam_m / adam_v float32 [K, P], step int32 [K], stats float64 [K, 4] on the device, each a view into a
    buffer with PAD sentinel elements before and after it."""

    def __init__(self, params, lr, active=None):
        K, P = params.shape
        self._raw = {}
        self.params = self._padded("params", params.float())
        self.m = self._padded("m", torch.zeros((K, P)))
        self.v = self._padded("v", torch.zeros((K, P)))
        self.step = self._padded("step", torch.zeros(K, dtype=torch.int32))
        self.stats = self._padded("stats", torch.zeros((K, 4), dtype=torch.float64))
        self.lr = torch.as_tensor(np.asarray(lr, np.float32)).cuda()
        self.active = (torch.ones(K, dtype=torch.uint8) if active is None else torch.as_tensor(active, dtype=torch.uint8)).cuda()

    def _padded(self, name, t):
        raw = torch.full((t.numel() + 2 * PAD,), SENTINEL, dtype=t.dtype).cuda()
        raw[PAD:PAD + t.numel()] = t.reshape(-1).cuda()
        self._raw[name] = raw
        return raw[PAD:PAD + t.numel()].view(t.shape)

    def sentinels_intact(self):
        return all(bool((r[:PAD] == SENTINEL).all()) and bool((r[-PAD:] == SENTINEL).all()) for r in self._raw.values())


def train_epoch(X, Y, bufs, train, val, L, A, batch):
    """One ovc_bc_train_epoch call: model k on the rows train[k] in that order, validated on val[k]."""
    K = len(train)
    stride = max([len(r) for r in list(train) + list(val)] + [1])
    tr = torch.zeros((K, stride), dtype=torch.int32)
    va = torch.zeros((K, stride), dtype=torch.int32)
    for k in range(K):
        tr[k, :len(train[k])] = torch.from_numpy(np.asarray(train[k], np.int32))
        va[k, :len(val[k])] = torch.from_numpy(np.asarray(val[k], np.int32))
    tr, va = tr.cuda(), va.cuda()
    nt = torch.tensor([len(r) for r in train], dtype=torch.int32).cuda()
    nv = torch.tensor([len(r) for r in val], dtype=torch.int32).cuda()
    lib = _bc_native.lib()
    _bc_native.check(lib.ovc_bc_train_epoch(
        X.data_ptr(), Y.data_ptr(), X.shape[0], tr.data_ptr(), nt.data_ptr(), va.data_ptr(), nv.data_ptr(), stride,
        bufs.params.data_ptr(), bufs.m.data_ptr(), bufs.v.data_ptr(), bufs.step.data_ptr(), bufs.lr.data_ptr(), bufs.active.data_ptr(),
        bufs.stats.data_ptr(), K, 96, 64, L, A, batch, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


# --- 1. against the float64 restatement ------------------------------------------------------------------------------

CONFIGS = [  # (hidden layers, actions, batch, training rows): every training set ends in a partial minibatch but the first
    dict(L=2, A=6, batch=64, n=320),
    dict(L=2, A=6, batch=64, n=300),
    dict(L=1, A=6, batch=64, n=300),
    dict(L=2, A=7, batch=1, n=90),
    dict(L=1, A=7, batch=128, n=300),
    dict(L=2, A=7, batch=128, n=300),
]


@pytest.mark.parametrize("epochs", [1, 3])
@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "L%d_A%d_b%d_n%d" % (c["L"], c["A"], c["batch"], c["n"]))
def test_epochs_match_the_float64_restatement(cfg, epochs):
    """The kernel's parameters, Adam moments, step, loss sums and correct counts after 1 and 3 epochs against the header's
    step restated in float64 on the same rows in the same order.

    The tolerance is float32's own rounding through the layers, measured on the same steps: the restatement also runs in
    float32 (torch on the CPU, another summation order than the kernel's FFMA chains), and each figure of the kernel may
    deviate from float64 by 8 times that restatement's largest deviation on the tensor, plus 16 units of float32 roundoff
    of the tensor's largest magnitude.  Two float32 evaluations of the same steps carry rounding errors of the same order
    but not of the same size, their summation orders being different.  A wrong step (another order of operations, a
    missing bias correction or 1/n) moves parameters by a share of lr per update, which the test checks to lie far
    above the tolerance.  Correct counts are exact but for rows whose two largest float64 logits lie within the logit
    tolerance, derived the same way."""
    L, A, batch, n = cfg["L"], cfg["A"], cfg["batch"], cfg["n"]
    _, X, Y = _golden_dataset()
    rng = np.random.RandomState(1000 * L + 100 * A + batch)
    Y = Y.clone()
    if A == 7:  # the seventh logit gets labels too
        Y[torch.from_numpy(rng.rand(Y.numel()) < 0.1).cuda()] = 6
    rows = rng.choice(X.shape[0], n + 40, replace=False)
    train, val = rows[:n], rows[n:]
    lr = 2e-3
    p0 = B.glorot_init(7, L, A)
    bufs = Buffers(p0[None], [lr])
    Xc, Yc = X.cpu(), Y.cpu().long()
    r64 = (p0.double(), torch.zeros_like(p0, dtype=torch.float64), torch.zeros_like(p0, dtype=torch.float64), 0)
    r32 = (p0, torch.zeros_like(p0), torch.zeros_like(p0), 0)
    for e in range(epochs):
        order = train[rng.permutation(n)]
        train_epoch(X, Y, bufs, [order], [val], L, A, batch)
        *r64, s64, z64 = ref_epoch(*r64, Xc, Yc, order, val, batch, L, A, lr, torch.float64)
        *r32, s32, z32 = ref_epoch(*r32, Xc, Yc, order, val, batch, L, A, lr, torch.float32)
        got = (bufs.params[0].cpu(), bufs.m[0].cpu(), bufs.v[0].cpu())
        for name, k, a, b in zip(("params", "adam_m", "adam_v"), got, r64[:3], r32[:3]):
            tol = 8 * float((b.double() - a).abs().max()) + 16 * U32 * float(a.abs().max())
            if name == "params":
                assert tol < lr / 10, "the tolerance %.3g no longer tells a wrong step from a right one" % tol
            dev = float((k.double() - a).abs().max())
            assert dev <= tol, (name, e, dev, tol)
        assert int(bufs.step[0]) == r64[3] == -(-n // batch) * (e + 1)
        st = bufs.stats[0].cpu().numpy()
        for i in (0, 2):
            tol = 8 * abs(s32[i] - s64[i]) + 16 * U32 * abs(s64[i])  # row losses are >= 0
            assert abs(st[i] - s64[i]) <= tol, (e, i, st[i], s64[i], tol)
        ztol = 8 * float((z32.double() - z64).abs().max()) + 16 * U32 * float(z64.abs().max())
        top2 = z64.topk(2, dim=1).values
        near = (top2[:, 0] - top2[:, 1] <= ztol).numpy()
        for i, part in ((1, slice(0, len(train))), (3, slice(len(train), None))):
            assert abs(st[i] - s64[i]) <= int(near[part].sum()), (e, i, st[i], s64[i], int(near[part].sum()))
    assert bufs.sentinels_intact()


# --- 2. independence -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [3, 200])
def test_models_of_one_launch_are_independent(K):
    """K models with different rows, seeds and lr give bit for bit what K launches of one model give; an inactive model's
    buffers are byte-identical afterwards, and no output is written outside its buffer."""
    _, X, Y = _golden_dataset()
    L, A, batch = 2, 6, 64
    rng = np.random.RandomState(K)
    sizes = rng.randint(1, 400, size=K)
    train = [rng.choice(X.shape[0], s, replace=False) for s in sizes]
    val = [rng.choice(X.shape[0], rng.randint(0, 100), replace=False) for _ in range(K)]
    lrs = rng.choice([1e-3, 3e-3, 5e-4], size=K)
    inits = torch.stack([B.glorot_init(100 + k, L, A) for k in range(K)])
    active = np.ones(K, np.uint8)
    active[K // 2] = 0  # one inactive model, its buffers garbage
    inits[K // 2] = torch.randn(inits.shape[1])
    bufs = Buffers(inits, lrs, active)
    for b in (bufs.m, bufs.v):
        b[K // 2] = torch.randn(inits.shape[1]).cuda()
    bufs.step[K // 2], bufs.stats[K // 2] = 12345, torch.tensor([1.5, 2.5, 3.5, 4.5])
    before = [t[K // 2].clone() for t in (bufs.params, bufs.m, bufs.v, bufs.step, bufs.stats)]
    orders = [[rng.permutation(r) for r in train] for _ in range(2)]
    for e in range(2):
        train_epoch(X, Y, bufs, orders[e], val, L, A, batch)
    assert bufs.sentinels_intact()
    for a, b in zip(before, (bufs.params, bufs.m, bufs.v, bufs.step, bufs.stats)):
        assert a.cpu().numpy().tobytes() == b[K // 2].cpu().numpy().tobytes()
    for k in range(K):
        if not active[k]:
            continue
        one = Buffers(inits[k:k + 1], lrs[k:k + 1])
        for e in range(2):
            train_epoch(X, Y, one, [orders[e][k]], [val[k]], L, A, batch)
        for a, b in ((one.params, bufs.params), (one.m, bufs.m), (one.v, bufs.v), (one.step, bufs.step), (one.stats, bufs.stats)):
            assert torch.equal(a[0], b[k]), k
        assert one.sentinels_intact()


# --- 3. the reference's greedy games ---------------------------------------------------------------------------------

def test_greedy_games_train_a_partner_that_plays():
    """The dataset of the reference's five GreedyHumanModel games is the golden featurize_state; train_bc with the
    reference's defaults beats the majority action on its training rows; the trained policy plays 400 transitions next to
    GreedyHumanModel through K10.  Accuracy and returns are printed, not asserted."""
    d, X, Y = _golden_dataset()
    assert torch.equal(X.cpu(), torch.from_numpy(d["feat_2"].reshape(-1, 96).astype(np.float32)))
    assert torch.equal(Y.cpu(), torch.from_numpy(d["actions"].reshape(-1).astype(np.int32)))
    models, hist = B.train_bc(X, Y, n_models=2, seeds=[0, 1])
    labels = d["actions"].reshape(-1)
    majority = np.bincount(labels).max() / labels.size
    for k, h in enumerate(hist):
        print("model %d: %d epochs, training accuracy %.4f (majority action %.4f), val accuracy %.4f, final lr %.1e"
              % (k, len(h["loss"]), h["accuracy"][-1], majority, h["val_accuracy"][-1], h["lr"][-1]))
        assert h["accuracy"][-1] > majority
        assert len(h["loss"]) <= 100 and all(np.isfinite(h["loss"]))
    env = BatchedOvercookedEnv("cramped_room", 256, horizon=400, auto_reset=True)
    pair = AgentPairRollout(env, (models[0], GreedyHumanModel()), seed=3)
    pair.run(400)
    fin = pair.episodes.finished()
    assert fin["env_index"].numel() == 256
    ret = fin["ep_sparse_r"].float()
    print("(BC, Greedy) on cramped_room: mean sparse return %.2f over %d episodes" % (float(ret.mean()), ret.shape[0]))
