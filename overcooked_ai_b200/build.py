"""Build csrc/libovc_b200.so, csrc/libovc_greedy.so, csrc/libovc_horizon.so and csrc/libovc_bc.so for the H100 (sm_90a) with nvcc, in-tree next to the sources.

    python -m overcooked_ai_b200.build [--force]
"""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["ovc_b200.cu"]
DEPS = ["ovc_b200.cu", "ovc_step.cuh", "ovc_obs.cuh", "ovc_encfc.cuh", "ovc_tail.cuh", "ovc_wide.cuh", "ovc_partner.cuh", "ovc_lstm.cuh", "ovc_potential.cuh", "ovc_potential_phi.inc", "ovc_rng.cuh", "ovc_host.cuh", "ovc_rollout.cuh", os.path.join("..", "..", "include", "ovc_b200.h")]
OUT = os.path.join(CSRC, "libovc_b200.so")
# the greedy partner's library (include/ovc_greedy.h): its own ABI, so the main library's exports and kernels stay as they are
GREEDY_SOURCES = ["ovc_greedy.cu"]
GREEDY_DEPS = ["ovc_greedy.cu", "ovc_rng.cuh", os.path.join("..", "..", "include", "ovc_b200.h"), os.path.join("..", "..", "include", "ovc_greedy.h")]
GREEDY_OUT = os.path.join(CSRC, "libovc_greedy.so")
# the horizon bootstrap's library (include/ovc_horizon.h): its own ABI too
HORIZON_SOURCES = ["ovc_horizon.cu"]
HORIZON_DEPS = ["ovc_horizon.cu", os.path.join("..", "..", "include", "ovc_b200.h"), os.path.join("..", "..", "include", "ovc_horizon.h")]
HORIZON_OUT = os.path.join(CSRC, "libovc_horizon.so")
# behaviour-cloning training (include/ovc_bc.h): its own ABI too
BC_SOURCES = ["ovc_bc.cu"]
BC_DEPS = ["ovc_bc.cu", os.path.join("..", "..", "include", "ovc_b200.h"), os.path.join("..", "..", "include", "ovc_bc.h")]
BC_OUT = os.path.join(CSRC, "libovc_bc.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return "nvcc"


def _compile(out, sources, deps, force, verbose, defines=()):
    newest = max(os.path.getmtime(os.path.join(CSRC, d)) for d in deps)
    if not force and os.path.exists(out) and os.path.getmtime(out) >= newest:
        return out
    cmd = [find_nvcc()] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + sources
    subprocess.check_call(cmd, cwd=CSRC)
    return out


def build(force=False, verbose=False, variant=None, defines=()):
    """Every library; returns the main one's path.  variant / defines: an experiment build of the main library only
    (csrc/libovc_b200_<variant>.so, compiled with the given -D macros); OVC_B200_LIB=<path> makes _native load it instead
    (tools/k5sweep.py A/B runs)."""
    if variant is not None:
        return _compile(os.path.join(CSRC, "libovc_b200_%s.so" % variant), SOURCES, DEPS, force, verbose, defines)
    _compile(GREEDY_OUT, GREEDY_SOURCES, GREEDY_DEPS, force, verbose)
    _compile(HORIZON_OUT, HORIZON_SOURCES, HORIZON_DEPS, force, verbose)
    _compile(BC_OUT, BC_SOURCES, BC_DEPS, force, verbose)
    return _compile(OUT, SOURCES, DEPS, force, verbose, defines)


if __name__ == "__main__":
    var = [a.split("=", 1)[1] for a in sys.argv if a.startswith("--variant=")]
    defs = [a[2:] for a in sys.argv if a.startswith("-D")]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=var[0] if var else None, defines=defs))
