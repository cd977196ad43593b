"""The table of policy-kernel instantiations in tests/test_gpu_policy_forms.py is what the built library holds: every
device instantiation of a policy-kernel template (K7, K8, the draw, K9, K11, K12) has a test that compares it with the
float64 restatement, so a new instantiation without one fails here."""
import ast
import os
import re
import shutil
import subprocess

import pytest

import test_gpu_policy_forms as F
from helpers import strip_signature
from overcooked_ai_b200 import _native

TESTS = os.path.dirname(os.path.abspath(__file__))
TEMPLATES = ("policy_tail_kernel", "policy_tail_grouped_kernel", "encode_linear_kernel", "encode_linear_masked_kernel",
             "encode_linear_grouped_kernel", "encode_linear_grouped_masked_kernel", "encode_linear_wgrad_kernel", "sample_actions_kernel",
             "wide_layers_kernel", "lstm_head_kernel")


def _tool(name):
    path = shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return path if os.path.exists(path) else None


def compiled_kernels():
    """The demangled names of every device entry point of the library, without return type and parameter list."""
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if not cuobjdump or not cufilt:
        pytest.skip("cuobjdump / cu++filt not installed: the compiled kernels cannot be listed")
    syms = subprocess.run([cuobjdump, "-symbols", _native.LIB_PATH], capture_output=True, text=True, check=True).stdout
    mangled = [line.split()[-1] for line in syms.splitlines() if "STO_ENTRY" in line]
    names = subprocess.run([cufilt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(names) == len(mangled) and len(set(names)) == len(names)
    return {strip_signature(n) for n in names}


def _compiled_policy_kernels():
    """The policy-kernel entry points, as ``ovc::<template><(args)>``."""
    pattern = re.compile(r"^ovc::(%s)<.*>$" % "|".join(TEMPLATES))
    return {n for n in compiled_kernels() if pattern.match(n)}


def test_every_policy_kernel_instantiation_has_a_float64_test():
    compiled = _compiled_policy_kernels()
    table = set(F.INSTANTIATIONS)
    untested, stale = sorted(compiled - table), sorted(table - compiled)
    assert not untested and not stale, ("compiled without an INSTANTIATIONS entry: %s; listed but not compiled: %s" % (untested, stale))
    print("%d policy-kernel instantiations, each with a float64 test" % len(compiled))


def defined_tests(module):
    with open(os.path.join(TESTS, module)) as f:
        tree = ast.parse(f.read())
    return {n.name for n in tree.body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}


def test_every_instantiation_names_a_test_that_exists():
    """An entry is a case of test_gpu_policy_forms.py (one of its test functions takes it) or names an existing test."""
    kinds = {"k8": "test_k8_form_exact", "k7": "test_k7_form_exact", "draw": "test_draw_form_exact", "k9": "test_k9_form_exact"}
    own = defined_tests("test_gpu_policy_forms.py")
    for name, entry in F.INSTANTIATIONS.items():
        if isinstance(entry, tuple):
            assert kinds[entry[0]] in own, (name, entry)
        else:
            module, test = entry.split("::")
            assert test in defined_tests(module), "%s names %s, which does not exist" % (name, entry)
