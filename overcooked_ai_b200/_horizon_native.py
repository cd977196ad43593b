"""ctypes binding of the C ABI in include/ovc_horizon.h (csrc/libovc_horizon.so): the horizon bootstrap's kernels.

Like ``_native``, no CPU fallback: a missing library or device raises.
"""
import ctypes
import os

from overcooked_ai_b200._native import NativeLibraryError

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libovc_horizon.so")

ABI_VERSION = 1
EXPORTED_SYMBOLS = ("ovc_horizon_abi_version", "ovc_horizon_last_error", "ovc_horizon_rows", "ovc_gae_horizon", "ovc_gae_horizon_view")

_lib = None


def lib():
    """Load (once) and return the horizon library; raises NativeLibraryError if it is not built or its ABI differs."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError("%s not found: the CUDA extension is not built (python -m overcooked_ai_b200.build). "
                                 "This engine has no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i64, f32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float
    L.ovc_horizon_abi_version.restype = ctypes.c_int
    L.ovc_horizon_last_error.restype = ctypes.c_char_p
    L.ovc_horizon_rows.argtypes = [vp, ctypes.c_int, vp, vp, ctypes.c_int, i64, vp, vp, vp, vp, vp, vp]
    L.ovc_horizon_rows.restype = ctypes.c_int
    for f in (L.ovc_gae_horizon, L.ovc_gae_horizon_view):
        f.argtypes = [vp, vp, vp, vp, vp, i64, i64, f32, f32, vp, vp, vp]
        f.restype = ctypes.c_int
    if L.ovc_horizon_abi_version() != ABI_VERSION:
        raise NativeLibraryError("ABI version mismatch: libovc_horizon %d, binding %d" % (L.ovc_horizon_abi_version(), ABI_VERSION))
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError("ovc horizon call failed (%d): %s" % (rc, lib().ovc_horizon_last_error().decode()))
