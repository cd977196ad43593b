"""Behaviour cloning on the device: the reference's ``train_bc_model`` (human_aware_rl/imitation/behavior_cloning_tf2.py) for
K models at once, from recorded games.

    feats, labels = bc_dataset(env, records, joint_actions)   # one row per (transition, player): its featurize view, its action
    models, history = train_bc(feats, labels, n_models=4, seeds=[0, 1, 2, 3])
    save_keras_npz(models[0], "bc.npz")                       # what examples/ppo_bc.py --bc-weights reads

Each epoch is one launch of ``ovc_bc_train_epoch`` (include/ovc_bc.h): one CTA per model runs every minibatch's forward
pass, backward pass and Adam update in float32 with the network in shared memory.  Between epochs the host runs the
reference's callbacks per model (``ReduceLROnPlateau`` and ``EarlyStopping`` on the training loss) on the epoch's four
figures, the one device sync per epoch.  The trained ``BCPolicy`` plays wherever a BC partner does; K10 rounds it to bf16
there (``BCPolicy.tables()``).  Recorded games in the reference's trajectory format enter through
``wire.records_from_dicts`` (states) and ``wire.action_indices`` (joint actions).
"""
import math

import numpy as np
import torch

from overcooked_ai_b200 import _bc_native
from overcooked_ai_b200.selfplay import BCPolicy

N_FEATURES, HIDDEN = 96, 64


def param_count(num_hidden_layers=2, num_actions=6):
    """P, the length of one model's flat parameter vector (include/ovc_bc.h)."""
    return N_FEATURES * HIDDEN + HIDDEN + (num_hidden_layers - 1) * (HIDDEN * HIDDEN + HIDDEN) + num_actions * HIDDEN + num_actions


def layer_shapes(num_hidden_layers=2, num_actions=6):
    """[(out, in)] of every layer in the flat vector's order: the hidden layers, then the logits."""
    dims = [N_FEATURES] + [HIDDEN] * num_hidden_layers
    return [(dims[i + 1], dims[i]) for i in range(num_hidden_layers)] + [(num_actions, HIDDEN)]


def glorot_init(seed, num_hidden_layers=2, num_actions=6):
    """A flat float32 parameter vector: Keras' default Dense initialisers, Glorot-uniform kernels (bound
    sqrt(6 / (fan_in + fan_out))) and zero biases, drawn from a CPU generator seeded with ``seed``."""
    g = torch.Generator().manual_seed(int(seed))
    parts = []
    for out, inp in layer_shapes(num_hidden_layers, num_actions):
        bound = math.sqrt(6.0 / (inp + out))
        parts += [(torch.rand((out, inp), generator=g, dtype=torch.float64) * 2 - 1).mul_(bound).float().reshape(-1),
                  torch.zeros(out)]
    return torch.cat(parts)


def policy_from_flat(flat, num_hidden_layers=2, num_actions=6):
    """A ``BCPolicy`` holding the flat vector (one copy; ``BCPolicy.parameters()`` is the flat order)."""
    pol = BCPolicy(num_hidden_layers=num_hidden_layers, num_actions=num_actions).to(flat.device)
    torch.nn.utils.vector_to_parameters(flat.detach().float(), pol.parameters())
    return pol


def validation_split_rows(n, split=0.15):
    """(train, val) positions of n rows as Keras' ``validation_split`` takes them: the last n - floor(n (1 - split)) rows
    are the validation rows, taken before any shuffle."""
    at = int(math.floor(n * (1.0 - split)))
    return np.arange(at), np.arange(at, n)


class KerasCallbacks(object):
    """The reference's callbacks on the training loss, for one model, run after each epoch in its order:
    ``ReduceLROnPlateau(monitor="loss", patience=3)`` (factor 0.1, min_delta 1e-4, cooldown 0, min_lr 0) and
    ``EarlyStopping(monitor="loss", patience=20)`` (min_delta 0).  ``lr`` is float32, as the optimizer's variable."""

    def __init__(self, lr, lr_patience=3, factor=0.1, min_delta=1e-4, stop_patience=20):
        self.lr = np.float32(lr)
        self.lr_patience, self.factor, self.min_delta, self.stop_patience = lr_patience, factor, min_delta, stop_patience
        self.lr_best, self.lr_wait = np.inf, 0
        self.stop_best, self.stop_wait = np.inf, 0

    def epoch_end(self, epoch, loss):
        """The training loss of epoch ``epoch`` (0-based) -> True when training stops after it; ``self.lr`` is the lr of
        the next epoch."""
        if loss < self.lr_best - self.min_delta:
            self.lr_best, self.lr_wait = loss, 0
        else:
            self.lr_wait += 1
            if self.lr_wait >= self.lr_patience and self.lr > 0:
                self.lr = np.float32(float(self.lr) * self.factor)
                self.lr_wait = 0
        self.stop_wait += 1
        if loss < self.stop_best:
            self.stop_best, self.stop_wait = loss, 0
            return False
        return self.stop_wait >= self.stop_patience and epoch > 0


def bc_dataset(env, records, joint_actions, num_pots=2):
    """Training rows from recorded games on ``env`` (its tables must hold the games' layouts): records int32 [M, S] (the
    state each joint action was taken in) and joint actions int [M, 2] -> (features float32 [2M, 96], labels int32 [2M]) on
    the device, row 2 i + p player p's featurize view of record i and its action."""
    recs = torch.as_tensor(np.asarray(records, dtype=np.int32) if not torch.is_tensor(records) else records).to(env.device, torch.int32)
    acts = torch.as_tensor(np.asarray(joint_actions) if not torch.is_tensor(joint_actions) else joint_actions).to(env.device, torch.int32)
    assert recs.dim() == 2 and acts.shape == (recs.shape[0], 2), "records [M, S] and joint actions [M, 2]"
    feats = env.featurize_state(num_pots=num_pots, states=recs.contiguous())
    return feats.reshape(-1, feats.shape[-1]), acts.reshape(-1).contiguous()


def train_bc(features, labels, n_models=1, rows=None, seeds=None, lr=1e-3, epochs=100, batch=64, validation_split=0.15,
             num_hidden_layers=2, num_actions=6, verbose=False):
    """Trains ``n_models`` BC models with the reference's recipe and returns ``(models, history)``.

    features float32 CUDA [R, 96], labels int32 CUDA [R] (``bc_dataset``).  Per model k: ``rows[k]`` (row indices into the
    dataset, default all rows; its last ``validation_split`` share, before any shuffle, validates), ``seeds[k]`` (default
    k: the Glorot init and the training rows' per-epoch shuffle on the device), ``lr`` (a float or one per model).
    ``models`` are ``BCPolicy`` on the device; ``history[k]`` is a dict of per-epoch lists ``loss``, ``accuracy``, ``val_loss``, ``val_accuracy`` (nan without
    validation rows) and ``lr`` (the lr the epoch ran with), as Keras' ``History`` holds them; a model that early
    stopping ends has fewer epochs."""
    lib = _bc_native.lib()
    dev = features.device
    assert features.is_cuda and features.dtype == torch.float32 and features.is_contiguous() and features.dim() == 2
    assert features.shape[1] == N_FEATURES, "features: featurize_state at num_pots = 2 (96 per row)"
    assert labels.is_cuda and labels.dtype == torch.int32 and labels.is_contiguous() and labels.numel() == features.shape[0]
    R, K = features.shape[0], int(n_models)
    lab_host = labels.cpu().numpy()
    assert ((lab_host >= 0) & (lab_host < num_actions)).all(), "labels must lie in [0, num_actions)"
    rows = [np.arange(R)] * K if rows is None else [np.asarray(r, dtype=np.int64) for r in rows]
    seeds = list(range(K)) if seeds is None else [int(s) for s in seeds]
    lrs = [float(lr)] * K if np.isscalar(lr) else [float(x) for x in lr]
    assert len(rows) == K and len(seeds) == K and len(lrs) == K
    for r in rows:
        assert r.ndim == 1 and ((r >= 0) & (r < R)).all(), "rows must index the dataset"
    splits = [validation_split_rows(len(r), validation_split) for r in rows]
    train = [torch.from_numpy(r[t].astype(np.int32)).to(dev) for r, (t, _) in zip(rows, splits)]
    stride = max([len(r) for r in rows] + [1])
    val_rows = torch.zeros((K, stride), dtype=torch.int32, device=dev)
    n_train = torch.tensor([len(t) for t, _ in splits], dtype=torch.int32, device=dev)
    n_val = torch.tensor([len(v) for _, v in splits], dtype=torch.int32, device=dev)
    for k, (r, (_, v)) in enumerate(zip(rows, splits)):
        val_rows[k, :len(v)] = torch.from_numpy(r[v].astype(np.int32)).to(dev)
    train_rows = torch.zeros((K, stride), dtype=torch.int32, device=dev)
    P = param_count(num_hidden_layers, num_actions)
    params = torch.stack([glorot_init(s, num_hidden_layers, num_actions) for s in seeds]).to(dev).contiguous()
    assert params.shape == (K, P)
    adam_m, adam_v = torch.zeros_like(params), torch.zeros_like(params)
    step = torch.zeros(K, dtype=torch.int32, device=dev)
    active = torch.ones(K, dtype=torch.uint8, device=dev)
    stats = torch.zeros((K, 4), dtype=torch.float64, device=dev)
    gens = [torch.Generator(device=dev).manual_seed(s) for s in seeds]
    cbs = [KerasCallbacks(x) for x in lrs]
    history = [dict(loss=[], accuracy=[], val_loss=[], val_accuracy=[], lr=[]) for _ in range(K)]
    live = np.ones(K, bool)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for epoch in range(int(epochs)):
        if not live.any():
            break
        for k in np.nonzero(live)[0]:  # the shuffle of the epoch, from the model's own generator
            n = len(train[k])
            train_rows[k, :n] = train[k][torch.randperm(n, generator=gens[k], device=dev)]
        lr_dev = torch.tensor([float(c.lr) for c in cbs], dtype=torch.float32).to(dev)
        _bc_native.check(lib.ovc_bc_train_epoch(
            features.data_ptr(), labels.data_ptr(), R, train_rows.data_ptr(), n_train.data_ptr(), val_rows.data_ptr(),
            n_val.data_ptr(), stride, params.data_ptr(), adam_m.data_ptr(), adam_v.data_ptr(), step.data_ptr(), lr_dev.data_ptr(),
            active.data_ptr(), stats.data_ptr(), K, N_FEATURES, HIDDEN, num_hidden_layers, num_actions, int(batch), stream))
        st = stats.cpu().numpy()
        for k in np.nonzero(live)[0]:
            nt, nv = len(splits[k][0]), len(splits[k][1])
            h = history[k]
            h["loss"].append(st[k, 0] / nt if nt else float("nan"))
            h["accuracy"].append(st[k, 1] / nt if nt else float("nan"))
            h["val_loss"].append(st[k, 2] / nv if nv else float("nan"))
            h["val_accuracy"].append(st[k, 3] / nv if nv else float("nan"))
            h["lr"].append(float(cbs[k].lr))
            if cbs[k].epoch_end(epoch, h["loss"][-1]):
                live[k] = False
                active[k] = 0
        if verbose:
            print("epoch %d: %d models training, loss %s" % (epoch, int(live.sum()), " ".join("%.4f" % h["loss"][-1] for h in history)))
    models = [policy_from_flat(params[k], num_hidden_layers, num_actions) for k in range(K)]
    return models, history


def keras_arrays(policy):
    """The Keras layout ``examples/ppo_bc.py --bc-weights`` reads: ``dense_<i>_kernel`` (in, out), ``dense_<i>_bias``,
    ``logits_kernel``, ``logits_bias``."""
    npy = lambda t: t.detach().float().cpu().numpy()
    out = {}
    for i, d in enumerate(policy.dense):
        out["dense_%d_kernel" % i], out["dense_%d_bias" % i] = npy(d.weight).T.copy(), npy(d.bias)
    out["logits_kernel"], out["logits_bias"] = npy(policy.logits.weight).T.copy(), npy(policy.logits.bias)
    return out


def save_keras_npz(policy, path):
    np.savez(path, **keras_arrays(policy))


def load_keras_npz(path):
    """A ``BCPolicy`` from ``save_keras_npz``'s file (or the reference's arrays in the same names)."""
    z = np.load(path)
    n_dense = len([k for k in z.files if k.startswith("dense_") and k.endswith("_kernel")])
    return BCPolicy(num_hidden_layers=n_dense, num_actions=z["logits_bias"].shape[0]).load_keras_weights(
        [(z["dense_%d_kernel" % i], z["dense_%d_bias" % i]) for i in range(n_dense)], (z["logits_kernel"], z["logits_bias"]))
