"""CPU tests of the C ABI binding: every prototype of include/centerpose_b200.h parses into the ctypes types the
library is called with, the built library exports and binds all of them, and the ctypes mirrors of the by-value
structs have the header's fields."""
import ctypes
import os
import re

import pytest

from centerpose_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


def test_every_prototype_parses():
    sigs = _lib.signatures()
    assert set(sigs) == set(re.findall(r"\b(cpb200_[a-z0-9_]+)\s*\(", HDR))
    queries = [n for n in sigs if n.endswith("_workspace_bytes")]
    assert len(queries) == 6
    for n in queries + ["cpb200_sizeof_op"]:
        assert sigs[n][0] is ctypes.c_size_t, n
    assert sigs["cpb200_version"] == (I, [])
    assert sigs["cpb200_last_error"] == (ctypes.c_char_p, [])
    assert sigs["cpb200_launch_count"] == (ctypes.c_ulonglong, [])
    assert sigs["cpb200_route_log_start"] == (None, [])
    assert sigs["cpb200_coco_kp_eval_workspace_bytes"][1] == [I, ctypes.c_int64, I, I, ctypes.c_int64]
    assert sigs["cpb200_soft_nms_39"] == (I, [P, I, F, F, F, I, P, P])
    assert sigs["cpb200_soft_nms_39_batch"] == (I, [P, I, I, F, F, F, I, P, P])
    H, T = _lib.Heads, _lib.Targets
    assert sigs["cpb200_multi_pose_loss_batch"] == (I, [H, T, I, I, P, P, P, P])
    assert sigs["cpb200_multi_pose_loss_train_batch"] == (I, [H, T, I, I, P, P, P, P, P])
    assert sigs["cpb200_multi_pose_loss_train_backward"] == (I, [H, T, I, I, P, P, P, H, P])
    for n in ("cpb200_multi_pose_targets_batch", "cpb200_multi_pose_targets_train_batch"):
        assert sigs[n] == (I, [P, I, P, I, T, P]), n


def test_multiline_prototype_with_comments_parses():
    text = """#define CPB200_X 1
    /* a comment with cpb200_not_a_function(int x); inside */
    size_t cpb200_a(int B,   /* batch */
                    int64_t n);
    typedef struct cpb200_s { int32_t a; } cpb200_s;
    unsigned long long cpb200_b(void);
    void cpb200_c(const double *m, double d, float f, void *stream);"""
    assert _lib.signatures(text) == {"cpb200_a": (ctypes.c_size_t, [I, ctypes.c_int64]),
                                     "cpb200_b": (ctypes.c_ulonglong, []),
                                     "cpb200_c": (None, [P, ctypes.c_double, F, P])}


@pytest.mark.parametrize("decl", ["int cpb200_x(long n, void *stream);", "uint32_t cpb200_x(void);",
                                  "int cpb200_x(cpb200_op op);", "cpb200_op cpb200_x(int n);"])
def test_unknown_type_raises(decl):
    with pytest.raises(TypeError, match=r"^cpb200_x: type '.+' has no ctypes binding"):
        _lib.signatures(decl)


def test_c_abi_exports_every_declared_symbol():
    L = _lib.lib()
    names = set(re.findall(r"\b(cpb200_[a-z0-9_]+)\s*\(", HDR))
    assert len(names) >= 9
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/centerpose_b200.h but not exported"
    for n, (restype, argtypes) in _lib.signatures().items():
        fn = getattr(L, n)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, n
    assert L.cpb200_version() >= 100
    from centerpose_b200.plan import OpStruct
    assert ctypes.sizeof(OpStruct) == L.cpb200_sizeof_op()
    assert L.cpb200_dcn_train_workspace_bytes(8, 64, 128, 128, 64) < 64 * 9 * 128 * 128 * 4
    assert L.cpb200_dcn_train_workspace_bytes(0, 64, 128, 128, 64) == 0


def _struct_fields(hdr, name):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = re.sub(r"\bconst\b", "", decl).strip()
        if decl:
            fields += [re.sub(r"[\s*]", "", f) for f in decl.split(None, 1)[1].replace("*", " ").split(",")]
    return fields


def test_c_abi_structs_and_signatures():
    for cls, name in ((_lib.Heads, "cpb200_multi_pose_heads"), (_lib.Targets, "cpb200_multi_pose_targets"),
                      (_lib.LossCfg, "cpb200_multi_pose_loss_cfg")):
        assert [f for f, _ in cls._fields_] == _struct_fields(HDR, name), name
    assert ctypes.sizeof(_lib.Heads) == 6 * 8 and ctypes.sizeof(_lib.Targets) == 11 * 8
    assert ctypes.sizeof(_lib.LossCfg) == 8 * 4
    for fn, n in (("cpb200_multi_pose_loss_train_batch", 9), ("cpb200_multi_pose_loss_train_backward", 9),
                  ("cpb200_multi_pose_loss_train_workspace_bytes", 1)):
        decl = re.search(r"\b%s\((.*?)\);" % fn, HDR, re.S).group(1)
        assert len(decl.split(",")) == n, fn
    if os.path.exists(_lib.LIBPATH):
        L = _lib.lib()
        assert L.cpb200_multi_pose_loss_train_workspace_bytes(32) == 8 * 3 * 18 * 32 + 4 * 6
