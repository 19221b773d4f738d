"""ctypes binding of the C ABI declared in ``include/centerpose_b200.h``.

The product path has NO CPU fallback: if the shared library is missing this module raises,
and every op raises ``RuntimeError`` on non-CUDA tensors.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBPATH = os.path.join(_HERE, "lib", "libcenterpose_b200.so")

_lib = None

c_float_p = ctypes.c_void_p   # raw device addresses are passed as integers


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIBPATH):
        raise RuntimeError(
            f"centerpose_b200: CUDA library not built ({LIBPATH} missing). Run "
            "`python -m centerpose_b200.build` (needs nvcc); there is no CPU fallback.")
    L = ctypes.CDLL(LIBPATH)
    L.cpb200_version.restype = ctypes.c_int
    L.cpb200_last_error.restype = ctypes.c_char_p
    L.cpb200_launch_count.restype = ctypes.c_ulonglong
    L.cpb200_decode_workspace_bytes.restype = ctypes.c_size_t
    L.cpb200_decode_workspace_bytes.argtypes = [ctypes.c_int] * 3
    L.cpb200_multi_pose_decode.restype = ctypes.c_int
    L.cpb200_multi_pose_decode.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int] * 6 + \
        [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.cpb200_multi_pose_decode_affine.restype = ctypes.c_int
    L.cpb200_multi_pose_decode_affine.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int] * 6 + \
        [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.cpb200_sigmoid_inplace.restype = ctypes.c_int
    L.cpb200_sigmoid_inplace.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    L.cpb200_flip_merge.restype = ctypes.c_int
    L.cpb200_flip_merge.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int), ctypes.c_void_p]
    L.cpb200_pre_process.restype = ctypes.c_int
    L.cpb200_pre_process.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.c_void_p,
                                     ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                                     ctypes.c_int, ctypes.c_void_p]
    L.cpb200_pre_process_batch.restype = ctypes.c_int
    L.cpb200_pre_process_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                                           ctypes.c_int, ctypes.c_void_p]
    L.cpb200_soft_nms_39.restype = ctypes.c_int
    L.cpb200_soft_nms_39.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                     ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    L.cpb200_soft_nms_39_batch.restype = ctypes.c_int
    L.cpb200_soft_nms_39_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                           ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    _lib = L
    return L


def check(status: int, what: str = "centerpose_b200"):
    if status != 0:
        msg = lib().cpb200_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what}: {msg} (status {status})")


def launch_count() -> int:
    return int(lib().cpb200_launch_count())
