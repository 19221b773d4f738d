"""Every device program the product lowers, pinned byte for byte: each (backbone, precision, size) plan is built on the
host and written out in a canonical text form whose SHA-256 must match ``tests/golden/plan_programs.json``.

The text holds every field of every ``cpb200_op`` but ``tc`` (the kernel's prepared state, filled at run time), each
``OP_HEADS`` table entry, the input / output slots and the activation bytes.  A pointer is written as what it points
into, so that addresses do not matter: an activation buffer (its index in ``Plan.buffers`` and the byte offset), a packed
weight or bias (the digest of its bytes and the byte offset), an external tensor (its name) or a head table.  A pointer
that resolves to none of these fails.

    python tests/test_plan_program_cpu.py            # regenerate the golden
    python tests/test_plan_program_cpu.py --texts D  # write each program's text to D/<config>.txt

With ``CPB200_PLAN_TEXTS=D`` holding texts written by the second command, a failure also names the first op and field
that differ.
"""
import ctypes
import hashlib
import json
import os
import sys

import pytest
import torch

ARCHS = ["dla_34", "res_50", "hrnet", "mobilenetv3", "hardnet", "mobilenetv2", "ghostnet"]
PRECISIONS = ["fp32", "bf16", "bf16x2", "fp16x2"]
SIZES = [(128, 160), (512, 512)]
B = 2
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plan_programs.json")
# environment switches that change what the builder emits
ENV = ("CPB200_RZ_COMP", "CPB200_S2D_STEM", "CPB200_NO_REUSE")


def configs():
    return [(a, p, h, w) for a in ARCHS for p in PRECISIONS for h, w in SIZES]


def key(arch, precision, H, W):
    return f"{arch}-{precision}-{H}x{W}"


def build_plan(arch, precision, H, W):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.model import create_model
    cfg = default_cfg(arch)
    torch.manual_seed(0)
    m = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg).set_precision(precision)
    return m._plan(B, H, W, torch.device("cpu"))


def _nbytes(t):
    return t.numel() * t.element_size()


class _Resolver:
    """pointer -> what it points into, as a stable string"""

    def __init__(self, plan):
        self.ranges = []                                   # (start, end, label, tensor or None)
        for i, b in enumerate(plan.buffers):
            self.ranges.append((b.data_ptr(), b.data_ptr() + _nbytes(b), f"buf{i}", None))
        for s in plan.pb.syms:
            if s.fixed and s.parent is None and s.buf is not None:
                self.ranges.append((s.buf.data_ptr(), s.buf.data_ptr() + _nbytes(s.buf), f"fixed:{s.name}", None))
        # smallest containing tensor first, so that a view kept beside its base resolves the same way every time
        for t in sorted(plan.pb.keep, key=_nbytes):
            self.ranges.append((t.data_ptr(), t.data_ptr() + _nbytes(t), None, t))
        self.tables = {ctypes.addressof(tab): f"heads@{i}" for i, tab in plan._head_tables.items()}
        self.digests = {}

    def __call__(self, p):
        if not p:
            return "null"
        if p in self.tables:
            return self.tables[p]
        for lo, hi, label, t in self.ranges:
            if lo <= p < hi:
                if label is None:
                    label = "w:" + self._digest(t)
                return f"{label}+{p - lo}"
        raise AssertionError(f"unresolved pointer {p:#x}")

    def _digest(self, t):
        d = self.digests.get(id(t))
        if d is None:
            raw = t.detach().contiguous().view(-1).view(torch.uint8).numpy()
            d = self.digests[id(t)] = f"{t.dtype}:{tuple(t.shape)}:" + hashlib.sha256(memoryview(raw)).hexdigest()[:20]
        return d


def program_text(plan) -> str:
    from centerpose_b200.plan import OpStruct
    res = _Resolver(plan)
    ptrs = {"src", "res", "aux", "dst", "weight", "bias"}
    lines = []
    for i in range(plan.n):
        o = plan.ops[i]
        fields = []
        for name, _ in OpStruct._fields_:
            if name == "tc":
                continue
            v = getattr(o, name)
            if name in ptrs:
                v = [res(e) for e in v] if name == "src" else res(v)
            elif name == "acc_scale":
                v = float(v).hex()
            elif not isinstance(v, int):
                v = list(v)
            fields.append(f"{name}={v}")
        lines.append(f"op{i} " + " ".join(fields))
    for i, tab in sorted(plan._head_tables.items()):
        for k, e in enumerate(tab):
            lines.append(f"op{i}.head{k} hidden={e.hidden} cout={e.cout} weight={res(e.weight)} bias={res(e.bias)} "
                         f"acc_scale3={float(e.acc_scale3).hex()} acc_scale1={float(e.acc_scale1).hex()}")
    lines.append(f"in_slots={plan.in_slots}")
    lines.append(f"out_slots={sorted(plan.out_slots.items())}")
    lines.append(f"buffers={[_nbytes(b) for b in plan.buffers]}")
    lines.append(f"activation_bytes={plan.activation_bytes}")
    return "\n".join(lines) + "\n"


def digest(text) -> str:
    return hashlib.sha256(text.encode()).hexdigest()


def _first_difference(old: str, new: str) -> str:
    for a, b in zip(old.splitlines(), new.splitlines()):
        if a != b:
            fa, fb = a.split(" "), b.split(" ")
            for x, y in zip(fa, fb):
                if x != y:
                    return f"{fa[0]}: {x} -> {y}"
            return f"{fa[0]}: {len(fa)} -> {len(fb)} fields"
    return f"{len(old.splitlines())} -> {len(new.splitlines())} lines"


def test_lowered_programs_match_golden(monkeypatch):
    for name in ENV:
        monkeypatch.delenv(name, raising=False)
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert sorted(golden) == sorted(key(*c) for c in configs())
    texts = os.environ.get("CPB200_PLAN_TEXTS")
    bad = []
    for c in configs():
        plan = build_plan(*c)
        text = program_text(plan)
        got, want = {"sha256": digest(text), "ops": plan.n}, golden[key(*c)]
        if got != want:
            msg = f"{key(*c)}: {want['ops']} ops -> {plan.n}"
            kept = os.path.join(texts, key(*c) + ".txt") if texts else None
            if kept and os.path.exists(kept):
                with open(kept) as f:
                    msg += ", first difference " + _first_difference(f.read(), text)
            bad.append(msg)
    assert not bad, f"{len(bad)} of {len(configs())} programs differ; first: {bad[0]}"


def main(argv):
    for name in ENV:
        os.environ.pop(name, None)
    texts = argv[argv.index("--texts") + 1] if "--texts" in argv else None
    out = {}
    for c in configs():
        plan = build_plan(*c)
        text = program_text(plan)
        out[key(*c)] = {"sha256": digest(text), "ops": plan.n}
        if texts:
            os.makedirs(texts, exist_ok=True)
            with open(os.path.join(texts, key(*c) + ".txt"), "w") as f:
                f.write(text)
        else:
            print(key(*c), out[key(*c)])
    if not texts:
        with open(GOLDEN, "w") as f:
            json.dump(out, f, indent=1, sort_keys=True)
            f.write("\n")


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    main(sys.argv[1:])
