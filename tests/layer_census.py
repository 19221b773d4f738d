"""Layer census: every layer call the backbone lowerings and the head make on ``PlanBuilder``, recorded from the real
lowering (``BackBoneWithHead._plan``) so that the op-level tests replay the shapes the models actually produce
(tests/test_layer_replay_gpu.py, tests/test_layer_census_cpu.py).  A helper module: it holds no tests.

A record is one OUTERMOST builder call: calls made inside another call (``deconv_k4s2`` -> four parity ``conv``,
``dcn`` -> its offset/mask conv, ``stem`` -> space-to-depth + conv, the CONVERT ops of fp32 islands) belong to the outer
call and are replayed through it.  ``REFERENCES`` holds a float64 torch evaluation of every recordable method.
"""
from __future__ import annotations

import functools
import inspect
import types
import zlib
from dataclasses import dataclass
from typing import Dict, List, Tuple

import pytest
import torch
import torch.nn.functional as F

ARCHS = ["dla_34", "res_50", "hrnet", "mobilenetv3", "hardnet", "mobilenetv2", "ghostnet"]

# public PlanBuilder methods that emit no op: symbols, views and finalisation.  Every other public method is recorded.
NOT_LAYERS = {"input", "output", "external", "keep_result", "channel_slice", "build"}
# arguments that carry the spatial size (dropped, with Sym H / W, from Record.shapeless)
SPATIAL_ARGS = {"Ho", "Wo", "out_map"}


@dataclass(frozen=True)
class Record:
    """method: PlanBuilder method name.  args: ((parameter, descriptor), ...) in signature order, defaults applied:
    a Sym is ("sym", C, H, W, kind, parent C or 0, channel offset), a tensor ("tensor", shape), a list a tuple of
    descriptors, anything else its value.  ops: (type, flags, act_dtype) of every op the call emitted."""
    method: str
    args: Tuple
    ops: Tuple

    @property
    def call(self) -> Tuple:
        return (self.method, self.args)

    @property
    def seed(self) -> int:
        """stable across processes and precisions (the same call replays the same data in every precision)"""
        return zlib.crc32(repr(self.call).encode())

    @property
    def shapeless(self) -> Tuple:
        return (self.method, tuple((k, _strip_hw(v)) for k, v in self.args if k not in SPATIAL_ARGS), self.ops)

    def arg(self, name):
        return dict(self.args)[name]

    def label(self) -> str:
        parts = []
        for k, v in self.args:
            if v is None or v is False or k in ("w", "b", "w_full", "om_w", "om_b"):
                continue
            parts.append(f"{k}={_short(v)}")
        w = dict(self.args).get("w", dict(self.args).get("w_full"))
        if w is not None:
            parts.insert(0, "w=" + "x".join(map(str, w[1])))
        ops = "/".join(f"{t}:{f}" for t, f, _ in self.ops)
        return f"{self.method}({', '.join(parts)}) ops[{ops}]"


def _short(v):
    if isinstance(v, tuple) and v and v[0] == "sym":
        _, C, H, W, kind, pc, off = v
        s = f"{C}@{H}x{W}" + ("" if kind == "act" else ":" + kind)
        return s + (f"[{off}:{off + C} of {pc}]" if pc else "")
    if isinstance(v, tuple) and v and isinstance(v[0], tuple):
        return "[" + ",".join(_short(e) for e in v) + "]"
    return repr(v)


def _strip_hw(v):
    if isinstance(v, tuple) and v and v[0] == "sym":
        return v[:2] + (None, None) + v[4:]
    if isinstance(v, tuple) and v and isinstance(v[0], tuple):
        return tuple(_strip_hw(e) for e in v)
    return v


def _desc(v):
    from centerpose_b200.plan import Sym
    if isinstance(v, Sym):
        return ("sym", v.C, v.H, v.W, v.kind, v.parent.C if v.parent is not None else 0, v.ch_off)
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape))
    if isinstance(v, (list, tuple)):
        return tuple(_desc(e) for e in v)
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    raise TypeError(f"layer census: cannot describe argument {v!r}")


def _recording(name):
    from centerpose_b200.plan import PlanBuilder
    base = getattr(PlanBuilder, name)
    sig = inspect.signature(base)

    @functools.wraps(base)
    def method(self, *args, **kw):
        if self._depth:
            return base(self, *args, **kw)
        start = len(self.ops)
        self._depth += 1
        try:
            out = base(self, *args, **kw)
        finally:
            self._depth -= 1
        bound = sig.bind(self, *args, **kw)
        bound.apply_defaults()
        desc = tuple((k, _desc(v)) for k, v in bound.arguments.items() if k != "self")
        self.records.append(Record(name, desc, tuple((int(o.type), int(o.flags), int(o.dtype)) for o in self.ops[start:])))
        self.spans.append((start, len(self.ops)))
        return out
    return method


@functools.lru_cache(maxsize=None)
def recording_builder_class():
    """PlanBuilder subclass that records every outermost public call and does not allocate a plan."""
    from centerpose_b200.plan import PlanBuilder

    def __init__(self, *a, **k):
        PlanBuilder.__init__(self, *a, **k)
        self.records: List[Record] = []
        self.spans: List[Tuple[int, int]] = []       # op index range [start, end) emitted by records[i]
        self._depth = 0

    def build(self):
        self.program = list(self.ops)                # the program before pruning
        return types.SimpleNamespace()

    ns = {"__init__": __init__, "build": build}
    for name, v in vars(PlanBuilder).items():
        if not name.startswith("_") and callable(v) and name not in NOT_LAYERS:
            ns[name] = _recording(name)
    return type("RecordingPlanBuilder", (PlanBuilder,), ns)


def lower_recorded(arch: str, precision: str, B: int, H: int, W: int):
    """Run the model's lowering (backbone + head) on a recording builder; returns the builder."""
    from centerpose_b200 import model as model_mod
    from centerpose_b200.config import default_cfg
    cfg = default_cfg(arch)
    m = model_mod.create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).set_precision(precision)
    made = []
    cls = recording_builder_class()

    def factory(*a, **k):
        pb = cls(*a, **k)
        made.append(pb)
        return pb
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(model_mod, "PlanBuilder", factory)
        m._plan(B, H, W, torch.device("cpu"))
    assert len(made) == 1
    return made[0]


@functools.lru_cache(maxsize=None)
def census(arch: str, precision: str, B: int, H: int, W: int) -> Tuple[Record, ...]:
    """the distinct layer calls of ``arch`` at (B, H, W) in ``precision``, in first-use order"""
    return tuple(dict.fromkeys(lower_recorded(arch, precision, B, H, W).records))


def signatures(arch: str, precision: str) -> List[Record]:
    """the calls the op-level replay runs: the census at 128x160, plus the 512x512 calls whose signature (spatial size
    ignored) the 128x160 census does not hold"""
    base = census(arch, precision, 1, 128, 160)
    seen = {r.shapeless for r in base}
    extra = [r for r in census(arch, precision, 1, 512, 512) if r.shapeless not in seen]
    return list(base) + list(dict.fromkeys(extra))


# ---------------------------------------------------------------------------------------- float64 references (NCHW)
def _act(y, act=None, relu=False):
    from oracle.mobilenet_ref import hsigmoid, hswish
    if act:
        return {"relu": F.relu, "hswish": hswish, "hsigmoid": hsigmoid, "relu6": lambda t: t.clamp(0, 6),
                "clip01": lambda t: t.clamp(0, 1)}[act](y)
    return F.relu(y) if relu else y


def _ref_conv(a):
    assert a["out_map"] is None, "strided-output convs are replayed through deconv_k4s2"
    # pad_hw = (top, left) of a conv without out_map pads bottom / right alike (PlanBuilder.conv's Ho / Wo)
    y = F.conv2d(torch.cat(a["srcs"], 1), a["w"], a["b"], stride=a["stride"],
                 padding=tuple(a["pad_hw"]) if a["pad_hw"] is not None else a["pad"])
    if a["res"] is not None:
        y = y + a["res"]
    return _act(y, a["act"], a["relu"])


def _ref_stem(a):
    return _act(F.conv2d(a["x"], a["w"], a["b"], stride=a["stride"], padding=a["pad"]), a["act"], a["relu"])


def _ref_deconv(a):
    # w_full is the BN-folded (Cout, Cin, 4, 4) weight of ConvTranspose2d(k4, s2, p1) in conv layout
    y = F.conv_transpose2d(a["x"], a["w_full"].transpose(0, 1), a["b"], stride=2, padding=1)
    return F.relu(y) if a["relu"] else y


def _ref_up_add(a):
    # PlanBuilder.up_add: act(conv_transpose2d(x, w, b, stride f, pad p, groups C)) + skip, f = stride or k // 2,
    # p = pad or f // 2
    C, _, k, _ = a["w"].shape
    f = k // 2 if a["stride"] is None else a["stride"]
    p = f // 2 if a["pad"] is None else a["pad"]
    y = _act(F.conv_transpose2d(a["x"], a["w"], a["b"], stride=f, padding=p, groups=C), a["act"])
    return y + a["skip"] if a["skip"] is not None else y


def _ref_dwconv(a):
    k = a["w"].shape[-1]
    return _act(F.conv2d(a["x"], a["w"], a["b"], stride=a["stride"], padding=k // 2, groups=a["x"].shape[1]), a["act"])


def _ref_scale_add(a):
    y = a["x"] * a["gate"]
    return y + a["skip"] if a["skip"] is not None else y


def _ref_upsample_add(a):
    y = F.interpolate(a["x"], scale_factor=a["f"], mode="nearest")
    if a["skip"] is not None:
        y = y + a["skip"]
    return F.relu(y) if a["relu"] else y


def _ref_dcn(a):
    from oracle import dcn_ref
    y = dcn_ref.dcn_module_forward(a["x"], a["w"], a["b"], a["om_w"], a["om_b"])
    return F.relu(y) if a["relu"] else y


REFERENCES: Dict[str, object] = {
    "conv": _ref_conv,
    "stem": _ref_stem,
    "deconv_k4s2": _ref_deconv,
    "maxpool": lambda a: F.max_pool2d(a["x"], a["k"], a["stride"], a["pad"]),
    "up_add": _ref_up_add,
    "dwconv": _ref_dwconv,
    "avgpool": lambda a: a["x"].mean(dim=(2, 3), keepdim=True),
    "scale_add": _ref_scale_add,
    "upsample_add": _ref_upsample_add,
    "avgpool2": lambda a: F.avg_pool2d(a["x"], 2, 2),
    "resize_bilinear": lambda a: F.interpolate(a["x"], size=(a["Ho"], a["Wo"]), mode="bilinear", align_corners=True),
    "dcn": _ref_dcn,
}
