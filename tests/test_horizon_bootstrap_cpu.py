"""The horizon bootstrap without a GPU: the library's header, exports, kernels and argument checks, and the configurations
collect(bootstrap_horizon=True) refuses."""
import ctypes
import os
import re
import subprocess
from types import SimpleNamespace

import pytest

import test_gpu_horizon_bootstrap as GH
from helpers import strip_signature
from overcooked_ai_b200 import _horizon_native
from overcooked_ai_b200.selfplay import AgentPairRollout, SelfPlayRollout
from test_policy_forms_cpu import _tool, defined_tests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_exports_agree():
    hdr = open(os.path.join(ROOT, "include", "ovc_horizon.h")).read()
    declared = set(re.findall(r"\b(ovc_(?:horizon|gae_horizon)[a-z_0-9]*)\s*\(", hdr))
    assert declared == set(_horizon_native.EXPORTED_SYMBOLS)
    lib = _horizon_native.lib()
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.ovc_horizon_abi_version() == _horizon_native.ABI_VERSION == int(re.search(r"OVC_HORIZON_ABI_VERSION (\d+)", hdr).group(1))


def test_library_kernels_are_the_gpu_tests_table():
    """Every device entry point of libovc_horizon.so has a case in tests/test_gpu_horizon_bootstrap.py, and every listed test
    exists."""
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if not cuobjdump or not cufilt:
        pytest.skip("cuobjdump / cu++filt not installed: the compiled kernels cannot be listed")
    syms = subprocess.run([cuobjdump, "-symbols", _horizon_native.LIB_PATH], capture_output=True, text=True, check=True).stdout
    mangled = [line.split()[-1] for line in syms.splitlines() if "STO_ENTRY" in line]
    names = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    assert {strip_signature(n) for n in names} == set(GH.KERNELS)
    own = defined_tests("test_gpu_horizon_bootstrap.py")
    for name, tests in GH.KERNELS.items():
        assert tests and set(tests) <= own, (name, tests)


def _buf():
    buf = (ctypes.c_int64 * 64)()
    return buf, ctypes.addressof(buf)


def test_rows_bad_arguments_are_refused():
    """Argument checks run before any launch, so they answer without a device."""
    lib = _horizon_native.lib()
    buf, p = _buf()
    ok = dict(state=p, state_words=16, done=p, partner_seat=None, one_view=0, n_envs=0, records=p, view=p, jrow=p, range=p, values=None,
              stream=None)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.ovc_horizon_rows(*[a[k] for k in ok]), lib.ovc_horizon_last_error().decode()

    assert call()[0] == 0  # nothing to do for n_envs = 0
    for kw, msg in ((dict(state=None), "null pointer"), (dict(range=None), "null pointer"), (dict(one_view=1), "partner_seat"),
                    (dict(n_envs=-1), "n_envs"), (dict(n_envs=1 << 30), "n_envs"), (dict(state_words=24), "state_words"),
                    (dict(state=p + 4), "aligned"), (dict(records=p + 8), "aligned"), (dict(jrow=p + 2), "aligned"),
                    (dict(values=p + 1), "aligned")):
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)


@pytest.mark.parametrize("fn", ["ovc_gae_horizon", "ovc_gae_horizon_view"])
def test_gae_bad_arguments_are_refused(fn):
    lib = _horizon_native.lib()
    buf, p = _buf()
    ok = dict(rewards=p, values=p, dones=p, terminal_values=p, last_values=p, n_steps=0, n=0, gamma=0.99, lam=0.95, adv=p, targets=p,
              stream=None)

    def call(**kw):
        a = dict(ok, **kw)
        return getattr(lib, fn)(*[a[k] for k in ok]), lib.ovc_horizon_last_error().decode()

    assert call()[0] == 0
    cases = [(dict(terminal_values=None), "null pointer"), (dict(adv=None), "null pointer"), (dict(n_steps=-1), "negative n_steps"),
             (dict(n=-2), "n_"), (dict(terminal_values=p + 2), "aligned")]
    if fn == "ovc_gae_horizon":
        cases += [(dict(n=3), "even"), (dict(rewards=p + 4), "8-byte aligned")]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc == -1 and msg in err, (kw, rc, err)


def _stub(cls, auto_reset=True, lstm=False, learners=None):
    """A rollout object with only what collect()'s refusals read: they come before any device work."""
    r = cls.__new__(cls)
    r.env = SimpleNamespace(auto_reset=auto_reset)
    if cls is SelfPlayRollout:
        r.lstm, r._learners = lstm, learners
    else:
        r.agents = [SimpleNamespace(lstm=lstm), SimpleNamespace(lstm=False)]
    return r


@pytest.mark.parametrize("cls", [SelfPlayRollout, AgentPairRollout], ids=["selfplay", "pair"])
def test_refused_configurations(cls):
    with pytest.raises(AssertionError, match="not supported for an LSTM learner"):
        _stub(cls, lstm=True).collect(8, 0.99, 0.95, bootstrap_horizon=True)
    with pytest.raises(AssertionError, match="bootstrap_horizon needs an auto_reset environment"):
        _stub(cls, auto_reset=False).collect(8, 0.99, 0.95, bootstrap_horizon=True)
    if cls is SelfPlayRollout:
        with pytest.raises(AssertionError, match="not supported for a population of learners"):
            _stub(cls, learners=object()).collect(8, 0.99, 0.95, bootstrap_horizon=True)
