"""ctypes binding of the C ABI in include/ovc_bc.h (csrc/libovc_bc.so): behaviour-cloning training.

Like ``_native``, no CPU fallback: a missing library or device raises.
"""
import ctypes
import os

from overcooked_ai_b200._native import NativeLibraryError

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libovc_bc.so")

ABI_VERSION = 1
MAX_BATCH = 128
EXPORTED_SYMBOLS = ("ovc_bc_abi_version", "ovc_bc_last_error", "ovc_bc_train_epoch")

_lib = None


def lib():
    """Load (once) and return the BC training library; raises NativeLibraryError if it is not built or its ABI differs."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError("%s not found: the CUDA extension is not built (python -m overcooked_ai_b200.build). "
                                 "This engine has no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    L.ovc_bc_abi_version.restype = ctypes.c_int
    L.ovc_bc_last_error.restype = ctypes.c_char_p
    L.ovc_bc_train_epoch.argtypes = [vp, vp, i64, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.ovc_bc_train_epoch.restype = ctypes.c_int
    if L.ovc_bc_abi_version() != ABI_VERSION:
        raise NativeLibraryError("ABI version mismatch: libovc_bc %d, binding %d" % (L.ovc_bc_abi_version(), ABI_VERSION))
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError("ovc bc call failed (%d): %s" % (rc, lib().ovc_bc_last_error().decode()))
