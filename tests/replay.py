"""Op-level replay machinery shared by tests/test_layer_replay_gpu.py and tests/test_kernel_envelope_gpu.py: one
``Record`` (tests/layer_census.py) run alone on the GPU with guarded output and poisoned inputs, its float64 reference,
and the per-precision bounds.  A helper module: it holds no tests.

Data (``_data``, seeded by the record's call):
  "f32" / "bf16": inputs randn (bf16-rounded in bf16); weights randn / sqrt(fan_in), bias and residual randn, DCN offset
           weights with gain 1.5 (as tests/test_split_gpu.py::test_dcn_split).
  "relu":  as "f32", with post-ReLU |randn| inputs to convs, dense deconvs and DCNs (the statistics plan.RZ_BETA was
           measured with).
  "int":   integer-exact data.  Activations in {-1, 0, 1}, bias in [-4, 4], weights sparse ternary with at most
           INT_NNZ nonzeros per output channel (depthwise filters: dense ternary).  Every product, partial sum and stored
           value is an integer of magnitude <= INT_NNZ + 5 (<= 256), so fp32, bf16 and fp16 hold each one exactly, even
           after fp16x2's 2^12 weight pre-scale (sums stay below 2^24 * 2^12 in steps of 2^12), the lo plane is 0 and the
           result equals the float64 reference bit for bit.  Needs CPB200_RZ_COMP=0 when the plan is built, so that
           acc_scale is a pure power of two.  The pools and the resize are exact on it where ``int_exact`` says so:
           means over 4 or 2^k pixels, and align-corners resizes whose weights are dyadic.
           DCN (_dcn_int): dyadic data.  x and the DCN weights / bias as above; the offset rows of om_w are sparse
           multiples of 1/4 with |w| <= 4 (exact in bf16, and under fp16x2's 2^12 pre-scale) and om_b's offsets
           multiples of 1/4, so every sampling position is a multiple of 1/4, exact in fp32 on every route; the mask
           rows of om_w are zero and the mask logits (om_b) exactly 0 or +-200, a mask of 0.5 or exactly 0 / 1 on every
           route.  Corner weights are multiples of 1/16, samples multiples of 1/32 with |s| <= 1 (at most 6 significant
           bits: the packed bf16 blend of the bf16 kernel is exact) and every output a multiple of 1/32 below 2^10 (15
           bits): the tensor-core sums and both split planes are exact, and each route equals the float64 reference as
           the output format stores it (_as_stored).
  "coord": a real-valued DCN with exact sampling positions (_dcn_coord).  x randn (bf16-rounded for bf16) except
           COORD_CH channels of small integers, which are the only channels the offset rows of om_w read (multiples of
           1/4, so with CPB200_RZ_COMP=0 the positions are exact and vary over space); mask rows randn.  Judged by the
           conv bounds (TOL), not the DCN's relative-L2 ones: only the arithmetic of the samples and the GEMM is left.

Tolerances (the op tests' bounds, tests/util.py::check_op; bf16 here is a max-norm, where check_op's is relative L2):
  fp32   : |err| <= 2e-4 max|ref|;  DCN 5e-4 (test_dcn_op_matches_oracle: the sampling positions come from the fp32
           offset conv, whose summation order differs from the reference's)
  bf16   : |err| <= 1e-2 max|ref|;  DCN relative L2 <= 2e-2
  bf16x2 : |err| <= 3e-4 max|ref|
  fp16x2 : |err| <= 1e-5 max|ref|
  split DCN: relative L2 <= 4 tol and |err| <= 40 tol max|ref|  (a sample within rounding of a pixel boundary flips corners)
  DCN on "coord" data: the conv bounds above (TOL)
  max-pool: exact on the values the input planes hold.
  "int" data: exact, element by element (against the reference as the output format stores it, RNE).

Guards.  Every check stays inside memory the test allocated.
  * Output canary: the final op(s) of the call write into [guard | output (both planes) | guard], all pre-filled with
    0xFF bytes (a NaN in every float format); afterwards the guards are unchanged and no output element still holds
    the pattern.  NCHW outputs get a destination with two spare channels on each side of their slice.
  * Input poison: every input and residual (both planes) sits at the front of an allocation whose tail is NaN, and a
    channel-slice input's parent holds NaN in every channel outside the slice, so a read outside an input shows up in
    the output: as NaN, or, where the ReLU epilogue or the fp16 saturation absorbs the NaN, as an error far above the
    bound.
"""
import math

import torch

from tests.layer_census import REFERENCES

DEV = "cuda:0"
TOL = {"fp32": 2e-4, "bf16": 1e-2, "bf16x2": 3e-4, "fp16x2": 1e-5}
DCN_TOL = {"fp32": 5e-4}
GUARD = 1 << 16                                  # bytes of canary on each side of an output
SENTINEL = 0xFF
WEIGHTS = {"w", "w_full", "om_w"}
BIASES = {"b", "om_b"}
RELU_INPUTS = {"conv": "srcs", "deconv_k4s2": "x", "dcn": "x"}
INT_NNZ = 96                                     # nonzeros per output channel of an integer-exact weight
# methods whose result is a sum of products of the inputs, weights and biases: "int" data makes them exact
INT_EXACT = {"conv", "stem", "deconv_k4s2", "maxpool", "up_add", "dwconv", "scale_add", "upsample_add", "avgpool",
             "avgpool2", "resize_bilinear", "dcn"}
MASK_LOGIT = (200.0, 0.0, -200.0)                # DCN "int" mask logits: sigmoid 1, 0.5 and 0 on every route
COORD_CH = 2                                     # DCN "coord": integer channels the offset rows read


def int_exact(rec):
    """whether ``rec`` has an exact leg on "int" data: a method of INT_EXACT without the h-swish / h-sigmoid activations
    (their /6 is not dyadic), an average pool over 2^k pixels, and an align-corners resize whose weights are dyadic:
    (Ho-1) / gcd(H-1, Ho-1) and the same ratio for W powers of two"""
    if rec.method not in INT_EXACT or dict(rec.args).get("act") in ("hswish", "hsigmoid"):
        return False
    if rec.method == "avgpool":
        _, _, H, W, _, _, _ = rec.arg("x")
        return (H * W) & (H * W - 1) == 0
    if rec.method == "resize_bilinear":
        _, _, H, W, _, _, _ = rec.arg("x")
        steps = [(o - 1) // math.gcd(i - 1, o - 1) for i, o in ((H, rec.arg("Ho")), (W, rec.arg("Wo")))]
        return all(s & (s - 1) == 0 for s in steps)
    return True


def _is_sym(d):
    return isinstance(d, tuple) and len(d) == 7 and d[0] == "sym"


def _is_syms(d):
    return isinstance(d, tuple) and len(d) > 0 and all(_is_sym(e) for e in d)


def _ternary(shape, g, nnz_per_row=None):
    """{-1, 0, 1} float32 tensor; with nnz_per_row, at most that many nonzeros in each row of dim 0"""
    t = torch.randint(-1, 2, shape, generator=g).float()
    n = t[0].numel()
    if nnz_per_row is None or n <= nnz_per_row:
        return t
    keep = torch.rand(shape[0], n, generator=g).argsort(1)[:, :nnz_per_row]
    sign = torch.randint(0, 2, keep.shape, generator=g).float() * 2 - 1
    return torch.zeros(shape[0], n).scatter_(1, keep, sign).reshape(shape)


def _quarters(shape, g, nnz, top=16):
    """sparse multiples of 1/4 with |w| <= top / 4: at most ``nnz`` nonzeros in each row of dim 0"""
    n = 1
    for s in shape[1:]:
        n *= s
    keep = torch.rand(shape[0], n, generator=g).argsort(1)[:, :nnz]
    q = torch.randint(1, top + 1, keep.shape, generator=g).float() / 4
    q *= torch.randint(0, 2, keep.shape, generator=g).float() * 2 - 1
    return torch.zeros(shape[0], n).scatter_(1, keep, q).reshape(shape)


def _dcn_int(rec, g, B):
    """dyadic DCN data (module docstring, "int").  Tap t's mask logit is MASK_LOGIT[(t + seed) % 3] (neighbouring taps
    differ).  Five of the six taps whose mask is not 0 are "near" taps: their offsets read only x channel 0, which is
    constant over each image (-1, 0, 1, -1, ...), so a near tap samples every pixel at one (dh, dw) per image, chosen
    so that its first sample row / column starts at a position of _DCN_START.  Over two images the five near taps take
    all nine (row start, column start) kinds of _DCN_START in turn, whose class sets (kernel_routes.DCN_CLASSES: p <= -1,
    (-1, 0), integer, fractional, (S-1, S), >= S) cross to every (h-class, w-class) pair.  The other taps read eight
    (channel, tap) entries of x with weights k/4, |k| <= 16, around a bias in [-6, 6]: positions that vary over the
    map, up to 38 pixels away."""
    x = rec.arg("x")
    C, H, W = x[1], x[2], x[3]
    co = rec.arg("w")[1][0]
    xs = _ternary((B, C, H, W), g)
    xs[:, 0] = (torch.arange(B) % 3 - 1).float().view(B, 1, 1)
    out = {"x": xs, "w": _ternary((co, C, 3, 3), g, INT_NNZ), "b": torch.randint(-4, 5, (co,), generator=g).float()}
    logits = [MASK_LOGIT[(t + rec.seed) % 3] for t in range(9)]
    near = [t for t in range(9) if logits[t] != MASK_LOGIT[2]][:5]
    om_w = torch.zeros(27, C, 3, 3)
    om_b = torch.zeros(27)
    kinds = [(h, w) for h in _DCN_START for w in _DCN_START]
    for t in range(9):
        if t not in near:
            om_w[2 * t:2 * t + 2] = _quarters((2, C, 3, 3), g, 8)
            om_b[2 * t:2 * t + 2] = torch.randint(-24, 25, (2,), generator=g).float() / 4
            continue
        k = near.index(t)
        d = []                                         # (dh, dw) of image 0 (x channel 0 = -1) and image 1 (= 0)
        for n in (0, 1):
            kh, kw = kinds[(5 * n + k) % 9]
            d.append((_DCN_START[kh][k % 2] - (t // 3 - 1), _DCN_START[kw][(k + n) % 2] - (t % 3 - 1)))
        for axis in (0, 1):
            om_b[2 * t + axis] = d[1][axis]
            om_w[2 * t + axis, 0, 1, 1] = d[1][axis] - d[0][axis]
    om_b[18:] = torch.tensor(logits)
    out["om_w"], out["om_b"] = om_w, om_b
    return out


# first sample position of a near tap's row or column (tap offset included), by kind: its classes on a map of size S
_DCN_START = {"below": (-1.25, -1.75),    # p <= -1, (-1, 0), fractional
              "above": (1.5, 1.25),       # fractional, (S-1, S), >= S
              "whole": (-1.0, 1.0)}       # p = -1, integers / integers, p = S


def _dcn_coord(rec, g, B, bf):
    """real-valued DCN data with exact sampling positions (module docstring, "coord")"""
    x = rec.arg("x")
    C, H, W = x[1], x[2], x[3]
    co = rec.arg("w")[1][0]
    rnd = (lambda t: t.bfloat16().float()) if bf else (lambda t: t)
    xs = torch.randn(B, C, H, W, generator=g)
    xs[:, :COORD_CH] = torch.randint(-3, 4, (B, COORD_CH, H, W), generator=g).float()
    om_w = torch.zeros(27, C, 3, 3)
    om_w[:18, :COORD_CH] = _quarters((18, COORD_CH, 3, 3), g, 4, top=8)
    om_w[18:] = rnd(torch.randn(9, C, 3, 3, generator=g) / (9 * C) ** 0.5)
    om_b = torch.zeros(27)
    om_b[:18] = torch.randint(-8, 9, (18,), generator=g).float() / 4
    om_b[18:] = torch.randn(9, generator=g)
    return {"x": rnd(xs), "w": rnd(torch.randn(co, C, 3, 3, generator=g) / (9 * C) ** 0.5),
            "b": torch.randn(co, generator=g), "om_w": om_w, "om_b": om_b}


def _data(rec, variant, B=2):
    """float32 CPU tensors for every tensor / Sym argument of ``rec`` (NCHW for Syms).  "coord" / "coord-bf16": DCN
    only (the latter bf16-rounded)."""
    g = torch.Generator().manual_seed(rec.seed)
    if variant in ("coord", "coord-bf16"):
        assert rec.method == "dcn", rec.method
        return _dcn_coord(rec, g, B, variant == "coord-bf16")
    if variant == "int" and rec.method == "dcn":
        return _dcn_int(rec, g, B)
    if variant == "int":
        out = {}
        for name, d in rec.args:
            if _is_sym(d) or _is_syms(d):
                ts = [None if s[4] == "nchw_out" else _ternary((B, s[1], s[2], s[3]), g)
                      for s in (d if _is_syms(d) else (d,))]
                out[name] = ts if _is_syms(d) else ts[0]
            elif isinstance(d, tuple) and len(d) == 2 and d[0] == "tensor":
                shape = d[1]
                if name in BIASES:
                    out[name] = torch.randint(-4, 5, shape, generator=g).float()
                elif rec.method in ("dwconv", "up_add"):
                    out[name] = _ternary(shape, g)
                else:
                    out[name] = _ternary(shape, g, INT_NNZ)
        return out
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
    B = pb.B
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


def _emit(pb, rec, data):
    """make ``rec``'s call on ``pb`` (inputs placed by _place_act) -> (result Sym, network-input buffer or None,
    output channel offset of an NCHW result or None)"""
    B = pb.B
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
    return getattr(pb, rec.method)(**kw), img_buf, ch_off


def _replay(rec, precision, data, guard_from_end=0, B=2, tc=None, run=None):
    """run ``rec`` alone on the GPU with guarded output and poisoned inputs -> (NCHW float64 result, guard problems).
    guard_from_end > 0 moves the start of the tail guard that many bytes into the output (the guards' own test).
    tc: PlanBuilder's tensor-core switch (False: bf16 on the CUDA-core kernels).  run(plan, stream) replaces
    plan.run (a profiler around it)."""
    from centerpose_b200.plan import PlanBuilder
    img = [d for _, d in rec.args if _is_sym(d) and d[4] == "nchw_in"]
    H, W = (img[0][2], img[0][3]) if img else (1, 1)
    pb = PlanBuilder(B, H, W, precision, torch.device(DEV), tc=tc)
    y, img_buf, ch_off = _emit(pb, rec, data)
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
    stream = torch.cuda.current_stream().cuda_stream
    if run is None:
        plan.run(stream)
    else:
        run(plan, stream)
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
    elif pb.split and y.kind == "act":
        planes = region.view(pb.torch16).view(shape).double()
        got = (planes[0] + planes[1]).permute(0, 3, 1, 2)
    else:
        got = region.view(torch.bfloat16 if esize == 2 else torch.float32).view(shape).double().permute(0, 3, 1, 2)
    if bool((bits == -1).any()):
        problems.append(f"left {int((bits == -1).sum())} output elements unwritten")
    if bool(got.isnan().any()):
        problems.append(f"{int(got.isnan().sum())} NaN outputs (read outside an input)")
    return got.cpu(), problems


def _as_stored(rec, precision, ref):
    """``ref`` rounded (RNE) to the format ``rec``'s result is stored in: fp32 (fp32 precision, fp32 / NCHW conv outputs,
    the split global average pool), bf16, or the sum of the two split planes"""
    from centerpose_b200.plan import split_planes
    f32 = precision == "fp32" or dict(rec.args).get("out", "act") != "act" or \
        (rec.method == "avgpool" and precision in ("bf16x2", "fp16x2"))
    if f32:
        return ref.float().double()
    if precision == "bf16":
        return ref.float().bfloat16().double()
    return split_planes(ref.float(), torch.float16 if precision == "fp16x2" else torch.bfloat16).double().sum(0)


def _judge(rec, precision, got, ref, exact=False, positions_exact=False):
    """-> (err / max|ref|, within bound, description).  positions_exact: a DCN on "coord" data, held to the conv bounds."""
    scale = ref.abs().max().item() + 1e-30
    diff = (got - ref).nan_to_num(float("inf")).abs()
    ratio = diff.max().item() / scale
    tol = TOL[precision]
    if exact:
        bad = int((got != _as_stored(rec, precision, ref)).sum())
        return ratio, bad == 0, f"exact: {bad} elements differ"
    if rec.method == "maxpool":
        return ratio, ratio == 0.0, "exact"
    if positions_exact:
        return ratio, ratio <= tol, f"tol {tol:.0e} (exact positions)"
    if rec.method == "dcn" and precision != "fp32":
        rel = ((got - ref).norm() / ref.norm()).item()
        if precision == "bf16":
            return ratio, rel <= 2e-2, f"relL2 {rel:.2e}"
        return ratio, rel <= 4 * tol and ratio <= 40 * tol, f"relL2 {rel:.2e}"
    if rec.method == "dcn":
        tol = DCN_TOL[precision]
    return ratio, ratio <= tol, f"tol {tol:.0e}"
