"""Behaviour-cloning training without a GPU: the library's header, exports and argument checks, the reference's callbacks
on synthetic loss curves, the validation split, the initialisation and the Keras weight file."""
import ctypes
import os
import re

import numpy as np
import torch

from overcooked_ai_b200 import _bc_native, bc as B
from overcooked_ai_b200.selfplay import BCPolicy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_exports_agree():
    hdr = open(os.path.join(ROOT, "include", "ovc_bc.h")).read()
    assert set(re.findall(r"\b(ovc_bc_[a-z_0-9]+)\s*\(", hdr)) == set(_bc_native.EXPORTED_SYMBOLS)
    lib = _bc_native.lib()
    for sym in _bc_native.EXPORTED_SYMBOLS:
        assert hasattr(lib, sym), sym
    assert lib.ovc_bc_abi_version() == _bc_native.ABI_VERSION == int(re.search(r"OVC_BC_ABI_VERSION (\d+)", hdr).group(1))
    assert _bc_native.MAX_BATCH == int(re.search(r"OVC_BC_MAX_BATCH (\d+)", hdr).group(1))


def test_param_count_is_the_headers_and_bcpolicys():
    assert B.param_count() == 10758
    for L in (1, 2):
        for A in (6, 7):
            assert B.param_count(L, A) == sum(p.numel() for p in BCPolicy(num_hidden_layers=L, num_actions=A).parameters())


def test_bad_arguments_are_refused():
    """Argument checks run before any launch, so they answer without a device."""
    lib = _bc_native.lib()
    buf = (ctypes.c_int64 * 64)()
    p = ctypes.addressof(buf)
    ok = dict(features=p, labels=p, n_rows=10, train_rows=p, n_train=p, val_rows=p, n_val=p, row_stride=10, params=p, adam_m=p,
              adam_v=p, step=p, lr=p, active=p, stats=p, n_models=0, n_features=96, hidden=64, num_hidden_layers=2, num_actions=6,
              batch=64, stream=None)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ovc_bc_train_epoch(*[a[k] for k in ok]), lib.ovc_bc_last_error().decode()

    assert call()[0] == 0  # nothing to do for n_models = 0
    assert call(active=p + 1)[0] == 0  # uint8 flags need no alignment
    for name in ("features", "labels", "train_rows", "n_train", "val_rows", "n_val", "params", "adam_m", "adam_v", "step", "lr",
                 "active", "stats"):
        assert call(**{name: None}) == (-1, call(**{name: None})[1]) and "null pointer" in call(**{name: None})[1], name
    for kw, msg in ((dict(n_models=-1), "negative n_models"), (dict(n_rows=-1), "n_rows"), (dict(n_rows=2**31), "n_rows"),
                    (dict(row_stride=-1), "row_stride"), (dict(row_stride=2**31), "row_stride"),
                    (dict(features=p + 4), "16-byte aligned"), (dict(stats=p + 4), "8-byte aligned")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)
    for name in ("labels", "train_rows", "n_train", "val_rows", "n_val", "params", "adam_m", "adam_v", "step", "lr"):
        rc, err = call(**{name: p + 2})
        assert rc == -1 and "4-byte aligned" in err, (name, rc, err)
    for kw, msg in ((dict(n_features=76), "n_features must be 96"), (dict(hidden=128), "hidden must be 64"),
                    (dict(num_hidden_layers=0), "num_hidden_layers"), (dict(num_hidden_layers=3), "num_hidden_layers"),
                    (dict(num_actions=1), "num_actions"), (dict(num_actions=8), "num_actions"), (dict(batch=0), "batch"),
                    (dict(batch=129), "batch")):
        rc, err = call(**kw)
        assert rc == -3 and msg in err, (kw, rc, err)
    assert call(batch=128, num_hidden_layers=1, num_actions=7)[0] == 0


def _run(losses, lr=1e-3):
    """Feeds a loss curve to the callbacks: (the epoch training stops after or None, the lr of every epoch run)."""
    cb = B.KerasCallbacks(lr)
    lrs = []
    for e, loss in enumerate(losses):
        lrs.append(float(cb.lr))
        if cb.epoch_end(e, loss):
            return e, lrs
    return None, lrs


def test_early_stopping_fires_twenty_epochs_after_the_last_improvement():
    stop, _ = _run([1.0] * 40)  # epoch 0 improves on inf, 1..20 do not
    assert stop == 20
    stop, _ = _run([1.0, 0.9, 0.8] + [0.8] * 30)  # last improvement at epoch 2 (equal is not an improvement)
    assert stop == 22
    stop, _ = _run([1.0 - 1e-9 * e for e in range(100)])  # any decrease improves (min_delta 0)
    assert stop is None


def test_lr_drops_after_three_epochs_within_min_delta():
    # epoch 0 sets the best; epochs 1-3 improve by less than 1e-4: the lr of epoch 4 is a tenth, then again from epoch 7
    curve = [1.0, 1.0 - 5e-5, 1.0 - 9e-5, 1.0 - 9.9e-5, 1.0 - 9.9e-5, 1.0 - 9.9e-5, 1.0 - 9.9e-5, 0.5]
    _, lrs = _run(curve)
    f32 = lambda x: float(np.float32(x))
    assert lrs == [f32(1e-3)] * 4 + [f32(f32(1e-3) * 0.1)] * 3 + [f32(f32(f32(1e-3) * 0.1) * 0.1)]
    # an improvement of more than min_delta resets the wait: no drop
    _, lrs = _run([1.0, 0.9998, 0.9996, 0.9994, 0.9992, 0.999])
    assert len(set(lrs)) == 1
    # the min_delta edge: 1.0 - 1e-4 - 2^-40 is an improvement, 1.0 - 1e-4 + 2^-40 is not
    cb = B.KerasCallbacks(1e-3)
    cb.epoch_end(0, 1.0)
    cb.epoch_end(1, 1.0 - 1e-4 - 2.0**-40)
    assert cb.lr_wait == 0 and cb.lr_best == 1.0 - 1e-4 - 2.0**-40
    cb = B.KerasCallbacks(1e-3)
    cb.epoch_end(0, 1.0)
    cb.epoch_end(1, 1.0 - 1e-4 + 2.0**-40)
    assert cb.lr_wait == 1 and cb.lr_best == 1.0


def test_validation_split_takes_the_last_rows_before_shuffling():
    for n, want in ((100, 15), (1000, 150), (7, 2), (4000, 600), (1, 1)):
        tr, va = B.validation_split_rows(n)
        assert len(va) == want
        assert np.array_equal(np.concatenate([tr, va]), np.arange(n))
    tr, va = B.validation_split_rows(20, 0.0)
    assert len(tr) == 20 and len(va) == 0


def test_glorot_init_bounds_and_reproducibility():
    for L, A in ((2, 6), (1, 7)):
        a, b, c = B.glorot_init(3, L, A), B.glorot_init(3, L, A), B.glorot_init(4, L, A)
        assert a.dtype == torch.float32 and a.numel() == B.param_count(L, A)
        assert torch.equal(a, b) and not torch.equal(a, c)
        pol = B.policy_from_flat(a, L, A)
        for (out, inp), lin in zip(B.layer_shapes(L, A), list(pol.dense) + [pol.logits]):
            bound = np.sqrt(6.0 / (inp + out))
            w = lin.weight.detach()
            assert w.shape == (out, inp) and float(w.abs().max()) <= bound and float(w.abs().max()) > 0.9 * bound
            assert abs(float(w.mean())) < 0.1 * bound and not lin.bias.detach().any()
        assert torch.equal(torch.nn.utils.parameters_to_vector(pol.parameters()), a)


def test_keras_npz_round_trip(tmp_path):
    for L, A in ((2, 6), (1, 7)):
        pol = B.policy_from_flat(B.glorot_init(11, L, A) + 0.01, L, A)
        path = str(tmp_path / ("bc_%d_%d.npz" % (L, A)))
        B.save_keras_npz(pol, path)
        z = np.load(path)
        assert sorted(z.files) == sorted(["dense_%d_%s" % (i, s) for i in range(L) for s in ("kernel", "bias")] + ["logits_kernel", "logits_bias"])
        assert z["dense_0_kernel"].shape == (96, 64) and z["logits_kernel"].shape == (64, A)
        n_dense = L
        back = BCPolicy(num_hidden_layers=n_dense, num_actions=A).load_keras_weights(
            [(z["dense_%d_kernel" % i], z["dense_%d_bias" % i]) for i in range(n_dense)], (z["logits_kernel"], z["logits_bias"]))
        for p, q in zip(pol.parameters(), back.parameters()):
            assert torch.equal(p, q)
        for p, q in zip(pol.parameters(), B.load_keras_npz(path).parameters()):
            assert torch.equal(p, q)
