"""Build csrc/libovc_b200.so for the H100 (sm_90a) with nvcc, in-tree next to the sources.

    python -m overcooked_ai_b200.build [--force]
"""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
SOURCES = ["ovc_b200.cu"]
DEPS = ["ovc_b200.cu", "ovc_step.cuh", "ovc_obs.cuh", "ovc_encfc.cuh", "ovc_tail.cuh", "ovc_wide.cuh", "ovc_potential.cuh", "ovc_rng.cuh", "ovc_host.cuh", "ovc_rollout.cuh", os.path.join("..", "..", "include", "ovc_b200.h")]
OUT = os.path.join(CSRC, "libovc_b200.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return "nvcc"


def build(force=False, verbose=False, variant=None, defines=()):
    """variant / defines: an experiment build next to the library (csrc/libovc_b200_<variant>.so, compiled with the given
    -D macros); OVC_B200_LIB=<path> makes _native load it instead (tools/k5sweep.py A/B runs)."""
    out = OUT if variant is None else os.path.join(CSRC, "libovc_b200_%s.so" % variant)
    newest = max(os.path.getmtime(os.path.join(CSRC, d)) for d in DEPS)
    if not force and os.path.exists(out) and os.path.getmtime(out) >= newest:
        return out
    cmd = [find_nvcc()] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    subprocess.check_call(cmd, cwd=CSRC)
    return out


if __name__ == "__main__":
    var = [a.split("=", 1)[1] for a in sys.argv if a.startswith("--variant=")]
    defs = [a[2:] for a in sys.argv if a.startswith("-D")]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, variant=var[0] if var else None, defines=defs))
