"""Op-level replay of every layer the five lowerings and the head produce (tests/layer_census.py), in all four
precisions, against a float64 torch evaluation of the same operation.

Which calls: the census of each arch at 128x160, replayed at the recorded spatial size, plus the 512x512 calls whose
signature (spatial size ignored) the 128x160 census does not hold.  B = 2, so the split kernels' "lo plane = batch
n + B" addressing is exercised.  Each call runs in a program of its own (the call's ops, plus the CONVERT ops an fp32
island adds around them).

Data (seeded by the record's call, so fp32 / bf16x2 / fp16x2 replay the same numbers and share one reference):
inputs randn (bf16-rounded in bf16); the split precisions replay every conv, dense deconv and DCN a second time with
post-ReLU |randn| inputs, the statistics plan.RZ_BETA was measured with.  Weights randn / sqrt(fan_in), bias and residual
randn, DCN offset weights with gain 1.5 (as tests/test_split_gpu.py::test_dcn_split).

Tolerances (those of tests/test_net_gpu.py, tests/test_split_gpu.py and tests/test_hardnet_gpu.py):
  fp32   : |err| <= 2e-4 max|ref|;  DCN 5e-4 (test_dcn_op_matches_oracle: the sampling positions come from the fp32
           offset conv, whose summation order differs from the reference's)
  bf16   : |err| <= 1e-2 max|ref|;  DCN relative L2 <= 2e-2
  bf16x2 : |err| <= 3e-4 max|ref|
  fp16x2 : |err| <= 1e-5 max|ref|
  split DCN: relative L2 <= 4 tol and |err| <= 40 tol max|ref|  (a sample within rounding of a pixel boundary flips corners)
  max-pool: exact on the values the input planes hold.  upsample_add always adds a skip here, whose sum is rounded
           (fp32, or re-split into planes), so it is held to the precision's bound.

Guards.  Every check stays inside memory this test allocated.
  * Output canary: the final op(s) of the call write into [guard | output (both planes) | guard], all pre-filled with
    0xFF bytes (a NaN in every float format); afterwards the guards are unchanged and no output element still holds
    the pattern.  NCHW outputs get a destination with two spare channels on each side of their slice.
  * Input poison: every input and residual (both planes) sits at the front of an allocation whose tail is NaN, and a
    channel-slice input's parent holds NaN in every channel outside the slice, so a read outside an input shows up in
    the output: as NaN, or, where the ReLU epilogue or the fp16 saturation absorbs the NaN, as an error far above the
    bound.
"""
import time

import pytest
import torch

from tests.layer_census import ARCHS, REFERENCES, census

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 2
TOL = {"fp32": 2e-4, "bf16": 1e-2, "bf16x2": 3e-4, "fp16x2": 1e-5}
DCN_TOL = {"fp32": 5e-4}
GUARD = 1 << 16                                  # bytes of canary on each side of an output
SENTINEL = 0xFF
WEIGHTS = {"w", "w_full", "om_w"}
BIASES = {"b", "om_b"}
RELU_INPUTS = {"conv": "srcs", "deconv_k4s2": "x", "dcn": "x"}
# fp32 / bf16x2 / fp16x2 replay identical data: keep them together so that they share the float64 references
PRECS = ["fp32", "bf16x2", "fp16x2", "bf16"]


def signatures(arch, precision):
    base = census(arch, precision, 1, 128, 160)
    seen = {r.shapeless for r in base}
    extra = [r for r in census(arch, precision, 1, 512, 512) if r.shapeless not in seen]
    return list(base) + list(dict.fromkeys(extra))


def _is_sym(d):
    return isinstance(d, tuple) and len(d) == 7 and d[0] == "sym"


def _is_syms(d):
    return isinstance(d, tuple) and len(d) > 0 and all(_is_sym(e) for e in d)


def _data(rec, variant):
    """float32 CPU tensors for every tensor / Sym argument of ``rec`` (NCHW for Syms)."""
    g = torch.Generator().manual_seed(rec.seed)
    bf = variant == "bf16"
    rnd = (lambda t: t.bfloat16().float()) if bf else (lambda t: t)
    relu_arg = RELU_INPUTS.get(rec.method) if variant == "relu" else None
    out = {}
    for name, d in rec.args:
        if _is_sym(d) or _is_syms(d):
            ts = []
            for s in (d if _is_syms(d) else (d,)):
                _, C, H, W, kind, _, _ = s
                if kind == "nchw_out":
                    ts.append(None)
                    continue
                t = torch.randn(B, C, H, W, generator=g)
                ts.append(rnd(t.abs() if name == relu_arg else t))
            out[name] = ts if _is_syms(d) else ts[0]
        elif isinstance(d, tuple) and len(d) == 2 and d[0] == "tensor":
            shape = d[1]
            t = torch.randn(*shape, generator=g)
            if name in BIASES:
                out[name] = t
            else:
                fan_in = 1
                for s in shape[1:]:
                    fan_in *= s
                out[name] = rnd(t * ((1.5 if name == "om_w" else 1.0) / fan_in ** 0.5))
    return out


def _reference(rec, data, stored=None):
    a = {k: v for k, v in rec.args}
    for k, v in (stored or data).items():
        if v is None:
            a[k] = None
        elif isinstance(v, list):
            a[k] = [t.double() for t in v]
        else:
            a[k] = v.double()
    return REFERENCES[rec.method](a)


def _stored(pb, t):
    """the values the activation planes of ``pb``'s precision hold for fp32 ``t``"""
    from centerpose_b200.plan import split_planes
    if pb.split:
        return split_planes(t, pb.torch16).double().sum(0)
    return t.double()


def _place_act(pb, t, d):
    """NCHW fp32 values -> an external activation at the front of a NaN-tailed allocation (a channel slice: inside a
    NaN-filled parent)."""
    # A NaN that is read does not always stay NaN: the ReLU epilogue (fmaxf) turns it into 0 and the fp16 planes'
    # saturation into -65504.  Every output channel of the pixel accumulates it, so the result is still far outside any
    # bound; the NaN count is the clearer message where it survives.
    from centerpose_b200.plan import split_planes
    _, C, H, W, kind, pc, off = d
    assert kind == "act", d
    cp = pc or C
    full = torch.full((B, H, W, cp), float("nan"))
    full[..., off:off + C] = t.permute(0, 2, 3, 1)
    if pb.split:
        data = split_planes(full, pb.torch16)               # (2, B, H, W, cp): hi plane, then lo plane
    else:
        data = full.to(pb.torch_act)
    n = data.numel()
    tail = max(4096, n // (B * (2 if pb.split else 1)))   # at least one image of one plane
    buf = torch.full((n + tail,), float("nan"), dtype=data.dtype, device=DEV)
    buf[:n] = data.reshape(-1).to(DEV)
    s = pb._sym(cp, H, W, "act", "external")
    s.fixed = True
    s.buf = buf
    return pb.channel_slice(s, off, C) if pc else s


def _replay(rec, precision, data, guard_from_end=0):
    """run ``rec`` alone on the GPU with guarded output and poisoned inputs -> (NCHW float64 result, guard problems).
    guard_from_end > 0 moves the start of the tail guard that many bytes into the output (the guards' own test)."""
    from centerpose_b200.plan import PlanBuilder
    img = [d for _, d in rec.args if _is_sym(d) and d[4] == "nchw_in"]
    H, W = (img[0][2], img[0][3]) if img else (1, 1)
    pb = PlanBuilder(B, H, W, precision, torch.device(DEV))
    kw, img_buf, ch_off = {}, None, None
    for name, d in rec.args:
        if _is_syms(d):
            kw[name] = [_place_act(pb, t, s) for t, s in zip(data[name], d)]
        elif _is_sym(d) and d[4] == "nchw_in":
            n = data[name].numel()
            img_buf = torch.full((n + max(4096, n // B),), float("nan"), device=DEV)
            img_buf[:n] = data[name].reshape(-1).to(DEV)
            kw[name] = pb.input(d[1])
        elif _is_sym(d) and d[4] == "nchw_out":
            kw[name] = pb.output(d[1] + 4, d[2], d[3], "out")        # two spare channels on each side of the slice
            ch_off = dict(rec.args)["ch_off"] + 2
        elif _is_sym(d):
            kw[name] = _place_act(pb, data[name], d)
        elif name in data:
            kw[name] = data[name]
        else:
            kw[name] = d
    if ch_off is not None:
        kw["ch_off"] = ch_off
    y = getattr(pb, rec.method)(**kw)
    if y.kind != "nchw_out":
        pb.keep_result(y)
    plan = pb.build()
    root = plan._root(y)
    last = [i for i, po in enumerate(plan.pb.ops) if plan._root(po.dst) is root]
    assert last, "the call's result has no producer"
    if y.kind == "nchw_out":
        esize, shape = 4, (B, y.C, y.H, y.W)
    elif y.kind == "act" and pb.split:
        esize, shape = 2, (2, B, y.H, y.W, y.C)
    elif y.kind == "act" and precision == "bf16":
        esize, shape = 2, (B, y.H, y.W, y.C)
    else:
        esize, shape = 4, (B, y.H, y.W, y.C)
    nbytes = esize
    for s in shape:
        nbytes *= s
    canary = torch.full((GUARD + nbytes + GUARD,), SENTINEL, dtype=torch.uint8, device=DEV)
    for i in last:
        plan.ops[i].dst = canary.data_ptr() + GUARD
    for (i, j) in plan.in_slots:
        plan.ops[i].src[j] = img_buf.data_ptr()
    plan.run(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    problems = []
    if not bool((canary[:GUARD] == SENTINEL).all()) or not bool((canary[GUARD + nbytes - guard_from_end:] == SENTINEL).all()):
        problems.append("wrote outside its output")
    region = canary[GUARD:GUARD + nbytes]
    bits = region.view(torch.int16 if esize == 2 else torch.int32).view(shape)
    if y.kind == "nchw_out":
        co = y.C - 4
        spare = torch.cat([bits[:, :ch_off], bits[:, ch_off + co:]], 1)
        if not bool((spare == -1).all()):
            problems.append("wrote outside its channel slice")
        bits = bits[:, ch_off:ch_off + co]
        got = region.view(torch.float32).view(shape)[:, ch_off:ch_off + co].double()
    elif pb.split:
        planes = region.view(pb.torch16).view(shape).double()
        got = (planes[0] + planes[1]).permute(0, 3, 1, 2)
    else:
        got = region.view(torch.bfloat16 if esize == 2 else torch.float32).view(shape).double().permute(0, 3, 1, 2)
    if bool((bits == -1).any()):
        problems.append(f"left {int((bits == -1).sum())} output elements unwritten")
    if bool(got.isnan().any()):
        problems.append(f"{int(got.isnan().sum())} NaN outputs (read outside an input)")
    return got.cpu(), problems


def _judge(rec, precision, got, ref):
    """-> (err / max|ref|, within bound, description)"""
    scale = ref.abs().max().item() + 1e-30
    diff = (got - ref).nan_to_num(float("inf")).abs()
    ratio = diff.max().item() / scale
    tol = TOL[precision]
    if rec.method == "maxpool":
        return ratio, ratio == 0.0, "exact"
    if rec.method == "dcn" and precision != "fp32":
        rel = ((got - ref).norm() / ref.norm()).item()
        if precision == "bf16":
            return ratio, rel <= 2e-2, f"relL2 {rel:.2e}"
        return ratio, rel <= 4 * tol and ratio <= 40 * tol, f"relL2 {rel:.2e}"
    if rec.method == "dcn":
        tol = DCN_TOL[precision]
    return ratio, ratio <= tol, f"tol {tol:.0e}"


_REF_CACHE = {"arch": None, "refs": {}}


def _cached_reference(arch, rec, variant, data):
    if _REF_CACHE["arch"] != arch:
        _REF_CACHE["arch"], _REF_CACHE["refs"] = arch, {}
    key = (rec.call, variant)
    if key not in _REF_CACHE["refs"]:
        _REF_CACHE["refs"][key] = _reference(rec, data)
    return _REF_CACHE["refs"][key]


@pytest.mark.parametrize("precision", PRECS)
def test_guards_notice_stray_writes_and_reads(precision):
    """The guards themselves, without touching memory outside this test's allocations: a tail guard that starts one
    pixel early must be reported as written, and a NaN planted in the last pixel of an input must reach the output."""
    rec = next(r for r in signatures("hardnet", precision) if r.method == "conv" and len(r.arg("srcs")) > 1)
    variant = "bf16" if precision == "bf16" else "f32"
    _, problems = _replay(rec, precision, _data(rec, variant))
    assert not problems, problems
    pixel = rec.arg("w")[1][0] * (2 if precision == "bf16" or precision.endswith("x2") else 4)
    _, problems = _replay(rec, precision, _data(rec, variant), guard_from_end=pixel)
    assert problems == ["wrote outside its output"], problems
    data = _data(rec, variant)
    ref = _reference(rec, data)
    data["srcs"][-1][-1, -1, -1, -1] = float("nan")
    got, problems = _replay(rec, precision, data)
    ratio, ok, _ = _judge(rec, precision, got, ref)
    assert not ok and ratio > 1e-2, (ratio, problems)


@pytest.mark.parametrize("arch,precision", [(a, p) for a in ARCHS for p in PRECS])
def test_layer_replay(arch, precision):
    t0 = time.time()
    recs = signatures(arch, precision)
    split = precision in ("bf16x2", "fp16x2")
    failures, worst, n = [], (-1.0, ""), 0
    for rec in recs:
        variants = ["bf16"] if precision == "bf16" else ["f32"]
        if split and rec.method in RELU_INPUTS:
            variants.append("relu")
        for variant in variants:
            n += 1
            label = f"{rec.label()} [{variant} inputs]"
            data = _data(rec, variant)
            try:
                got, problems = _replay(rec, precision, data)
            except Exception as e:                          # an op the library rejects is a finding too
                failures.append(f"{label}: {type(e).__name__}: {e}")
                continue
            if rec.method == "maxpool":
                from centerpose_b200.plan import PlanBuilder
                pb = PlanBuilder(B, 1, 1, precision, torch.device("cpu"))
                ref = _reference(rec, data, {"x": _stored(pb, data["x"])})
            elif variant == "bf16":
                ref = _reference(rec, data)
            else:
                ref = _cached_reference(arch, rec, variant, data)
            ratio, ok, how = _judge(rec, precision, got, ref)
            if ratio > worst[0]:
                worst = (ratio, label)
            if problems or not ok:
                failures.append(f"{label}: err/max {ratio:.3e} ({how}){'; ' + '; '.join(problems) if problems else ''}")
    print(f"\n{arch} {precision}: {len(recs)} signatures, {n} replays, worst err/max {worst[0]:.3e} at {worst[1]}"
          f" ({time.time() - t0:.1f} s)")
    assert not failures, f"{arch} {precision}: {len(failures)} of {n} replays failed:\n" + "\n".join(failures)
