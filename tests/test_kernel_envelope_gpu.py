"""Every network-op kernel route at the edges of the shapes its dispatcher accepts (tests/kernel_routes.py CASES and
HEAD_CASES), against a float64 evaluation of the same operation, with the replay guards of tests/replay.py.

Each case runs twice where it can:
  * integer-exact data (tests/replay.py "int"): the result must equal the reference bit for bit, element by element, in
    every precision, so a dropped, doubled or shifted tap, K slab, tile row / column, padding error or wrong channel
    offset fails whatever the format's rounding (CPB200_RZ_COMP=0 at plan build: acc_scale a pure power of two);
  * randn data under the per-precision bounds of the layer replay (rounding, the hi / lo split, the RZ compensation).
    hswish / hsigmoid and the global average pools over sizes that are not powers of two take this leg only.
DCN cases take the exact leg on dyadic data (exact sampling positions; the result equals the reference as the output
format rounds it) and a third, "coord" leg between the two: real-valued samples at exact positions, held to the conv
bounds, so a split gather that loses the lo plane fails where the DCN's own loose randn bounds would pass it.
The first leg also runs with the library's route log on: the set of kernels the program launched must equal the case's
route set.
"""
import time

import pytest
import torch

from tests.kernel_routes import CASES, HEAD_CASES, heads_program, kernel_key
from tests.replay import DEV, GUARD, SENTINEL, TOL, _data, _judge, _place_act, _reference, _replay, _stored

pytestmark = pytest.mark.gpu
WORST = {}                                        # precision -> (worst err / max|ref| on randn data, case)


def _precision(p):
    """case precision key -> (PlanBuilder precision, tensor-core switch)"""
    return ("bf16", False) if p == "bf16-simt" else (p, None)


def _launched(plan, stream, names):
    """plan.run with the library's route log on (cpb200_route_log_start / _read): adds the kernels it launched,
    normalised, to ``names``.  The log is read, and recording stopped, even when the run fails."""
    import ctypes
    from centerpose_b200 import _lib
    L = _lib.lib()
    L.cpb200_route_log_start()
    try:
        plan.run(stream)
        torch.cuda.synchronize()
    finally:
        buf = ctypes.create_string_buffer(1 << 16)
        n = L.cpb200_route_log_read(buf, len(buf))
        if n < 0:
            raise RuntimeError(f"route_log_read: {L.cpb200_last_error().decode()}")
        names.update(kernel_key(k) for k in buf.value.decode().splitlines() if k)


def _note(precision, ratio, label):
    if ratio > WORST.get(precision, (-1.0, ""))[0]:
        WORST[precision] = (ratio, label)


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    print(f"\nkernel envelope: {time.time() - t0:.1f} s; worst err/max on randn data:")
    for p, (r, label) in sorted(WORST.items()):
        print(f"  {p:10s} {r:.3e}  {label}")


@pytest.mark.parametrize("idx,pkey", [(i, p) for i, c in enumerate(CASES) for p in c.precisions()],
                         ids=[f"{i}-{p}-{c.rec.method}" for i, c in enumerate(CASES) for p in c.precisions()])
def test_route(idx, pkey, monkeypatch):
    case = CASES[idx]
    precision, tc = _precision(pkey)
    want = case.routes_for(pkey)
    names = set()
    if case.error:
        with pytest.raises(RuntimeError, match=case.error):
            _replay(case.rec, precision, _data(case.rec, "f32", case.B), B=case.B, tc=tc,
                    run=lambda plan, st: _launched(plan, st, names))
        assert names == set(), names
        return
    bf = precision == "bf16"
    coord = ["coord-bf16" if bf else "coord"] if case.rec.method == "dcn" else []
    legs = (["int"] if case.exact else []) + coord + ["bf16" if bf else "f32"]
    failures = []
    for leg in legs:
        data = _data(case.rec, leg, case.B)
        with monkeypatch.context() as mp:
            if leg == "int" or leg in coord:
                mp.setenv("CPB200_RZ_COMP", "0")
            got, problems = _replay(case.rec, precision, data, B=case.B, tc=tc,
                                    run=(lambda plan, st: _launched(plan, st, names)) if leg == legs[0] else None)
        if leg == legs[0] and names != set(want):
            failures.append(f"launched {sorted(names)}, declared {sorted(want)}")
        if case.rec.method == "maxpool" and leg != "int":
            from centerpose_b200.plan import PlanBuilder
            pb = PlanBuilder(case.B, 1, 1, precision, torch.device("cpu"))
            ref = _reference(case.rec, data, {"x": _stored(pb, data["x"])})
        else:
            ref = _reference(case.rec, data)
        ratio, ok, how = _judge(case.rec, precision, got, ref, exact=leg == "int", positions_exact=leg in coord)
        if leg != "int":
            _note(pkey, ratio, case.label())
        if problems or not ok:
            failures.append(f"[{leg}] err/max {ratio:.3e} ({how}){'; ' + '; '.join(problems) if problems else ''}")
    assert not failures, f"{case.label()} {pkey}:\n" + "\n".join(failures)


# ------------------------------------------------------------------------------------------------------------ heads
def _head_params(hc, leg, g):
    """per head (w3, b3, w1, b1) fp32 CPU tensors.  "int": hidden <= 8 + 4 in magnitude, outputs <= 16 * 12 + 4."""
    from tests.replay import _ternary
    out = []
    for co in hc.couts:
        if leg == "int":
            w3 = _ternary((hc.hid, hc.C, 3, 3), g, 8)
            w1 = _ternary((co, hc.hid, 1, 1), g, 16)
            b3 = torch.randint(-4, 5, (hc.hid,), generator=g).float()
            b1 = torch.randint(-4, 5, (co,), generator=g).float()
        else:
            w3 = torch.randn(hc.hid, hc.C, 3, 3, generator=g) / (9 * hc.C) ** 0.5
            w1 = torch.randn(co, hc.hid, 1, 1, generator=g) / hc.hid ** 0.5
            b3, b1 = torch.randn(hc.hid, generator=g), torch.randn(co, generator=g)
            if leg == "bf16":
                w3, w1 = w3.bfloat16().float(), w1.bfloat16().float()
        out.append((w3, b3, w1, b1))
    return out


def _heads_run(hc, precision, x, params, names=None):
    """-> ([NCHW float64 result per head], guard problems)"""
    from centerpose_b200 import plan as plan_mod
    pb = plan_mod.PlanBuilder(hc.B, hc.H, hc.W, precision, torch.device(DEV))
    xs = _place_act(pb, x, ("sym", hc.C, hc.H, hc.W, "act", 0, 0))
    outs = [pb.output(co, hc.H, hc.W, f"head{k}") for k, co in enumerate(hc.couts)]
    heads_program(pb, xs, params, outs)
    plan = pb.build()
    fused = [o for o in plan.pb.ops if o.type == plan_mod.OP_HEADS]
    assert len(fused) == 1 and len(fused[0].heads) == hc.fused, [o.type for o in plan.pb.ops]
    canaries, views = [], {}
    for k, co in enumerate(hc.couts):
        nbytes = hc.B * co * hc.H * hc.W * 4
        c = torch.full((GUARD + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
        canaries.append((c, nbytes))
        views[f"head{k}"] = c[GUARD:GUARD + nbytes].view(torch.float32)
    plan.bind(None, views)
    stream = torch.cuda.current_stream().cuda_stream
    if names is None:
        plan.run(stream)
    else:
        _launched(plan, stream, names)
    torch.cuda.synchronize()
    got, problems = [], []
    for k, ((c, nbytes), co) in enumerate(zip(canaries, hc.couts)):
        if not bool((c[:GUARD] == SENTINEL).all()) or not bool((c[GUARD + nbytes:] == SENTINEL).all()):
            problems.append(f"head {k}: wrote outside its output")
        bits = c[GUARD:GUARD + nbytes].view(torch.int32)
        if bool((bits == -1).any()):
            problems.append(f"head {k}: left {int((bits == -1).sum())} output elements unwritten")
        got.append(c[GUARD:GUARD + nbytes].view(torch.float32).view(hc.B, co, hc.H, hc.W).double().cpu())
    return got, problems


def _heads_reference(pb_like, x, params):
    """float64 conv1x1(relu(conv3x3(x))), the hidden map rounded as the precision stores it"""
    import torch.nn.functional as F
    out = []
    for w3, b3, w1, b1 in params:
        h = F.relu(F.conv2d(x.double(), w3.double(), b3.double(), padding=1))
        if pb_like.precision == "bf16":
            h = h.float().bfloat16().double()
        else:
            h = _stored(pb_like, h.float())
        out.append(F.conv2d(h, w1.double(), b1.double()))
    return out


@pytest.mark.parametrize("idx,precision", [(i, p) for i, c in enumerate(HEAD_CASES) for p in c.precisions()])
def test_heads(idx, precision, monkeypatch):
    from centerpose_b200.plan import PlanBuilder
    hc = HEAD_CASES[idx]
    pb_like = PlanBuilder(hc.B, 1, 1, precision, torch.device("cpu"))
    failures = []
    for leg in ("int", "bf16" if precision == "bf16" else "f32"):
        g = torch.Generator().manual_seed(1000 + idx)
        if leg == "int":
            x = torch.randint(-1, 2, (hc.B, hc.C, hc.H, hc.W), generator=g).float()
        else:
            x = torch.randn(hc.B, hc.C, hc.H, hc.W, generator=g)
            if leg == "bf16":
                x = x.bfloat16().float()
        params = _head_params(hc, leg, g)
        names = set() if leg == "int" else None
        with monkeypatch.context() as mp:
            if leg == "int":
                mp.setenv("CPB200_RZ_COMP", "0")
            got, problems = _heads_run(hc, precision, x, params, names)
        if names is not None and names != set(hc.routes_for(precision)):
            failures.append(f"launched {sorted(names)}, declared {sorted(hc.routes_for(precision))}")
        refs = _heads_reference(pb_like, x, params)
        for k, (gk, rk) in enumerate(zip(got, refs)):
            diff = (gk - rk).nan_to_num(float("inf")).abs()
            ratio = diff.max().item() / (rk.abs().max().item() + 1e-30)
            if leg == "int":
                ok = bool((diff == 0).all())
            else:
                ok = ratio <= TOL[precision]
                _note(precision, ratio, f"{hc.label()} head {k}")
            if not ok:
                failures.append(f"[{leg}] head {k} (cout {hc.couts[k]}): err/max {ratio:.3e}, "
                                f"{int((diff != 0).sum())} of {diff.numel()} elements differ")
        failures += [f"[{leg}] {p}" for p in problems]
    assert not failures, f"{hc.label()} {precision}:\n" + "\n".join(failures)
