"""ctypes binding of the C ABI declared in ``include/centerpose_b200.h``.

The header is the only statement of the ABI: ``lib()`` binds ``restype`` and ``argtypes`` of every ``cpb200_*``
prototype from it when the library loads, and a type the binding does not know fails the load.  ``launch`` makes
every call that enqueues work on a stream; the queries that take none (``*_workspace_bytes``, ``launch_count``,
``sizeof_op``, ``prepare_ops``, ``release_ops``) are plain calls on ``lib()``.

The product path has NO CPU fallback: if the shared library is missing this module raises,
and every op raises ``RuntimeError`` on non-CUDA tensors.
"""
from __future__ import annotations

import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBPATH = os.path.join(_HERE, "lib", "libcenterpose_b200.so")
HEADER = os.path.join(_HERE, "..", "include", "centerpose_b200.h")

_lib = None


class Targets(ctypes.Structure):
    """``cpb200_multi_pose_targets``: the device addresses of the eleven target arrays."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("hm", "hm_hp", "wh", "reg", "ind", "reg_mask", "hps", "hps_mask",
                                               "hp_offset", "hp_ind", "hp_mask")]


class Heads(ctypes.Structure):
    """``cpb200_multi_pose_heads``: the device addresses of the six head maps."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset")]


class LossCfg(ctypes.Structure):
    """``cpb200_multi_pose_loss_cfg``."""
    _fields_ = [(n, ctypes.c_float) for n in ("hm_weight", "wh_weight", "off_weight", "hp_weight", "hm_hp_weight")] + \
               [(n, ctypes.c_int32) for n in ("hm_hp", "reg_offset", "reg_hp_offset")]


# the by-value types of the header; every pointer is bound as c_void_p (device addresses are passed as integers,
# host arrays as ctypes arrays or byref), a `const char *` return as c_char_p
_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
          "double": ctypes.c_double, "unsigned long long": ctypes.c_ulonglong,
          "cpb200_multi_pose_heads": Heads, "cpb200_multi_pose_targets": Targets}
_PROTOTYPE = re.compile(r"(.+?)\b(cpb200_\w+)\s*\((.*)\)", re.S)


def _ctype(fn: str, decl: str, ret: bool):
    """The ctypes type of ``fn``'s return type or parameter declaration ``decl``."""
    words = [w for w in decl.replace("*", " * ").split() if w != "const"]
    if "*" in words:
        return ctypes.c_char_p if ret and words == ["char", "*"] else ctypes.c_void_p
    t = " ".join(words)
    if ret and t == "void":
        return None
    if not ret and t not in _TYPES:
        t = " ".join(words[:-1])           # drop the parameter's name
    if t not in _TYPES:
        raise TypeError(f"{fn}: type {decl.strip()!r} has no ctypes binding (include/centerpose_b200.h)")
    return _TYPES[t]


def signatures(text: str | None = None) -> dict:
    """``{name: (restype, argtypes)}`` of every ``cpb200_*`` prototype of ``text`` (default: the header).  Reads no
    library, so it also works where the library is not built."""
    if text is None:
        with open(HEADER) as f:
            text = f.read()
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", " ", text, flags=re.M)
    sigs = {}
    for stmt in re.split(r"[;{}]", text):
        m = _PROTOTYPE.fullmatch(stmt.strip())
        if m:
            ret, name, params = m.groups()
            params = [p for p in params.split(",") if p.strip() not in ("", "void")]
            sigs[name] = (_ctype(name, ret, True), [_ctype(name, p, False) for p in params])
    return sigs


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIBPATH):
        raise RuntimeError(
            f"centerpose_b200: CUDA library not built ({LIBPATH} missing). Run "
            "`python -m centerpose_b200.build` (needs nvcc); there is no CPU fallback.")
    L = ctypes.CDLL(LIBPATH)
    for name, (restype, argtypes) in signatures().items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


def check(status: int, what: str = "centerpose_b200"):
    if status != 0:
        msg = lib().cpb200_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what}: {msg} (status {status})")


def launch(name: str, device, *args) -> None:
    """``cpb200_<name>(*args, stream)`` with ``device``'s current stream, inside a device guard.  Tensors are passed as
    their ``data_ptr()`` and None as NULL; a non-zero status raises ``RuntimeError`` naming the entry point."""
    fn = getattr(lib(), "cpb200_" + name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(device):
        st = fn(*args, torch.cuda.current_stream(device).cuda_stream)
    check(st, "cpb200_" + name)


def launch_count() -> int:
    return int(lib().cpb200_launch_count())
