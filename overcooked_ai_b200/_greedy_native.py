"""ctypes binding of the C ABI in include/ovc_greedy.h (csrc/libovc_greedy.so): the greedy partner's kernel.

Like ``_native``, no CPU fallback: a missing library or device raises.
"""
import ctypes
import os

from overcooked_ai_b200._native import NativeLibraryError

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libovc_greedy.so")

ABI_VERSION = 1
EXPORTED_SYMBOLS = ("ovc_greedy_abi_version", "ovc_greedy_layout_table_size", "ovc_greedy_last_error", "ovc_greedy_actions")

_lib = None


def lib():
    """Load (once) and return the greedy library; raises NativeLibraryError if it is not built or its ABI differs."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError("%s not found: the CUDA extension is not built (python -m overcooked_ai_b200.build). "
                                 "This engine has no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp = ctypes.c_void_p
    L.ovc_greedy_abi_version.restype = ctypes.c_int
    L.ovc_greedy_layout_table_size.restype = ctypes.c_size_t
    L.ovc_greedy_last_error.restype = ctypes.c_char_p
    L.ovc_greedy_actions.argtypes = [vp, vp, vp, ctypes.c_int, vp, vp, vp, vp, ctypes.c_int64, ctypes.c_int, ctypes.c_uint64, vp, vp, vp]
    L.ovc_greedy_actions.restype = ctypes.c_int
    if L.ovc_greedy_abi_version() != ABI_VERSION:
        raise NativeLibraryError("ABI version mismatch: libovc_greedy %d, binding %d" % (L.ovc_greedy_abi_version(), ABI_VERSION))
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError("ovc greedy call failed (%d): %s" % (rc, lib().ovc_greedy_last_error().decode()))
