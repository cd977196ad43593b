"""Every device entry point of the built library has a reference test: each is a key of exactly one of the two tables,
tests/test_gpu_policy_forms.py::INSTANTIATIONS (the policy kernels, against the float64 restatement) and
tests/test_gpu_env_forms.py::INSTANTIATIONS (every other kernel, against the CPU oracle or its restatement), so a new
kernel or template instantiation without one fails here."""
import test_gpu_env_forms as E
import test_gpu_policy_forms as F
from test_policy_forms_cpu import compiled_kernels, defined_tests


def test_every_kernel_instantiation_is_in_exactly_one_table():
    compiled = compiled_kernels()
    env, policy = set(E.INSTANTIATIONS), set(F.INSTANTIATIONS)
    assert not env & policy, sorted(env & policy)
    untested, stale = sorted(compiled - env - policy), sorted((env | policy) - compiled)
    assert not untested and not stale, ("compiled without an INSTANTIATIONS entry: %s; listed but not compiled: %s" % (untested, stale))
    print("%d device entry points: %d policy-kernel and %d environment-kernel instantiations" % (len(compiled), len(policy), len(env)))


def test_every_environment_instantiation_names_a_test_that_exists():
    """An entry is a K1 / K5 case of test_gpu_env_forms.py (one of its test functions takes it) or names an existing test."""
    kinds = {"k1": ["test_k1_form_vs_oracle"], "k5": ["test_k5_form_vs_oracle", "test_k5_form_with_the_prefetch_vs_oracle"]}
    own = defined_tests("test_gpu_env_forms.py")
    for name, entry in E.INSTANTIATIONS.items():
        if isinstance(entry, tuple):
            assert set(kinds[entry[0]]) <= own, (name, entry)
        else:
            module, test = entry.split("::")
            assert test in defined_tests(module), "%s names %s, which does not exist" % (name, entry)
