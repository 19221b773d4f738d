"""CPU checks of the DCN cases of tests/kernel_routes.py and of their data (tests/replay.py):

  * the dyadic ("int") data meets every premise that makes each route's result exact, on the cases and on every DCN
    signature the backbones record; the "coord" data keeps its sampling positions exact;
  * each constructed case reaches the sampling classes it claims (kernel_routes.DCN_CLASSES, per axis), and together
    the cases reach every (h-class, w-class) pair on each DCN kernel family and launch every reachable DCN kernel;
  * the data discriminates: the float64 reference differs from seven plausible gather bugs (BUGS), restated here;
  * oracle.dcn_ref's vectorised reference equals its literal loops on the small cases (exactly -1, S-1 and S included);
  * the library refuses a DCN whose 32-bit gather offsets would overflow, before it allocates or launches anything.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from tests.kernel_routes import CASES, DCN_CLAIMS, ROUTES, UNREACHABLE
from tests.layer_census import ARCHS, census
from tests.replay import COORD_CH, INT_NNZ, MASK_LOGIT, _data, _reference

DCN = [(i, c) for i, c in enumerate(CASES) if c.rec.method == "dcn"]
BUGS = ("swap dh / dw", "mask of tap t + 1", "mask of tap t - 1", "trunc for floor", "h_high < H-1", "w_high < W-1",
        "every sample from image 0")
DCN_CLASSES_H = ("<=-1", "(-1,0)", "int", "frac", "(S-1,S)", ">=S")     # short names of kernel_routes.DCN_CLASSES


def _ids(cases):
    return [f"{i}-{c.rec.arg('x')[1]}x{c.rec.arg('x')[2]}x{c.rec.arg('x')[3]}-co{c.rec.arg('w')[1][0]}-B{c.B}"
            for i, c in cases]


def _census_dcn():
    out = {}
    for arch in ARCHS:
        for size in ((128, 160), (512, 512)):
            for r in census(arch, "fp32", 1, *size):
                if r.method == "dcn":
                    out.setdefault(r.call, r)
    return list(out.values())


def _d(data):
    return {k: v.double() for k, v in data.items()}


def _field(x, om_w, om_b, bug=None):
    """float64 sampling field of a DCN -> (ph, pw, mask, dh, dw), each (B, 9, H, W): tap t samples x at
    (h - 1 + t // 3 + dh, w - 1 + t % 3 + dw) with weight mask"""
    B, C, H, W = x.shape
    om = F.conv2d(x, om_w, om_b, padding=1)
    dh, dw = om[:, 0:18:2], om[:, 1:18:2]
    if bug == "swap dh / dw":
        dh, dw = dw, dh
    mask = torch.sigmoid(om[:, 18:27])
    if bug == "mask of tap t + 1":
        mask = mask.roll(-1, 1)
    elif bug == "mask of tap t - 1":
        mask = mask.roll(1, 1)
    tap = torch.arange(9, dtype=torch.float64)
    ph = torch.arange(H, dtype=torch.float64).view(1, 1, H, 1) + (tap // 3 - 1).view(1, 9, 1, 1) + dh
    pw = torch.arange(W, dtype=torch.float64).view(1, 1, 1, W) + (tap % 3 - 1).view(1, 9, 1, 1) + dw
    return ph, pw, mask, dh, dw


def _columns(x, om_w, om_b, bug=None):
    """float64 sampled columns (B, C, 9, H*W): mask * bilinear sample, dcn_v2_im2col's arithmetic, or one bug's"""
    B, C, H, W = x.shape
    ph, pw, mask, _, _ = _field(x, om_w, om_b, bug)
    rnd = torch.trunc if bug == "trunc for floor" else torch.floor
    h0, w0 = rnd(ph), rnd(pw)
    lh, lw = ph - h0, pw - w0
    hmax = H - 2 if bug == "h_high < H-1" else H - 1
    wmax = W - 2 if bug == "w_high < W-1" else W - 1
    inside = (ph > -1) & (pw > -1) & (ph < H) & (pw < W)
    flat = x.reshape(B, C, H * W)
    if bug == "every sample from image 0":
        flat = flat[:1].expand(B, C, H * W)
    col = torch.zeros(B, C, 9 * H * W, dtype=torch.float64)
    for hy, wx, wt, ok in ((h0, w0, (1 - lh) * (1 - lw), (h0 >= 0) & (w0 >= 0)),
                           (h0, w0 + 1, (1 - lh) * lw, (h0 >= 0) & (w0 + 1 <= wmax)),
                           (h0 + 1, w0, lh * (1 - lw), (h0 + 1 <= hmax) & (w0 >= 0)),
                           (h0 + 1, w0 + 1, lh * lw, (h0 + 1 <= hmax) & (w0 + 1 <= wmax))):
        ok = ok & inside
        idx = (hy.clamp(0, H - 1) * W + wx.clamp(0, W - 1)).long().reshape(B, 1, 9 * H * W)
        col += flat.gather(2, idx.expand(B, C, 9 * H * W)) * (wt * ok).reshape(B, 1, 9 * H * W)
    return col.reshape(B, C, 9, H * W) * mask.reshape(B, 1, 9, H * W)


def _dcn64(d, relu=True, bug=None):
    x = d["x"]
    B, C, H, W = x.shape
    col = _columns(x, d["om_w"], d["om_b"], bug)
    co = d["w"].shape[0]
    y = torch.einsum("okt,bktn->bon", d["w"].reshape(co, C, 9), col) + d["b"].view(1, co, 1)
    y = y.reshape(B, co, H, W)
    return F.relu(y) if relu else y


def _classes(p, S):
    """per-axis sampling class (index into kernel_routes.DCN_CLASSES) of every position"""
    c = torch.full(p.shape, -1, dtype=torch.long)
    whole = p == p.floor()
    c[p <= -1] = 0
    c[(p > -1) & (p < 0)] = 1
    c[(p >= 0) & (p <= S - 1) & whole] = 2
    c[(p > 0) & (p < S - 1) & ~whole] = 3
    c[(p > S - 1) & (p < S)] = 4
    c[p >= S] = 5
    assert (c >= 0).all()
    return c


def _reach(case, d):
    """-> (the DCN_CLAIMS the data reaches, the set of (h-class, w-class) pairs on taps whose mask is not 0)"""
    x = d["x"]
    B, C, H, W = x.shape
    ph, pw, mask, dh, dw = _field(x, d["om_w"], d["om_b"])
    live = mask > 1e-30                          # a logit of -200: mask 0 on the device
    ch, cw = _classes(ph, H), _classes(pw, W)
    pairs = set(zip(ch[live].tolist(), cw[live].tolist()))
    got = set()
    if len(pairs) == 36:
        got.add("all-pairs")
    TW = 16 if W >= 16 else 8
    TH = 128 // TW
    inside = (ph >= 0) & (ph <= H - 1) & (pw >= 0) & (pw <= W - 1)
    if bool((live & inside & (dh.abs() > TH)).any()) and bool((live & inside & (dw.abs() > TW)).any()):
        got.add("beyond-tile")
    if bool((live & ((dh.abs() > H) | (dw.abs() > W))).any()):
        got.add("beyond-map")
    values = [set(mask[:, t][live[:, t]].unique().tolist()) | ({0.0} if not bool(live[:, t].all()) else set())
              for t in range(9)]
    if all(sum(v in vs for vs in values) >= 2 for v in (0.0, 0.5, 1.0)):
        got.add("masks")
    last = live[-1] & (ph[-1] > H - 2) & (ph[-1] < H) & (pw[-1] > W - 2) & (pw[-1] < W)
    if B >= 2 and bool(last.any()):
        got.add("last-pixel")
    return got, pairs


def _family(pkey, kernel):
    """the DCN kernel family of a launched kernel, or None"""
    if kernel.startswith("conv_tc_kernel<") and ",true," in kernel:
        return f"tensor-core P = {kernel[-2]}"
    if kernel.startswith("conv_simt_kernel<") and kernel.endswith(",true>"):
        return "split fp32 island" if pkey == "x2" else "CUDA-core"
    return None


@pytest.fixture(scope="module")
def reached():
    out = {}
    for i, c in DCN:
        out[i] = _reach(c, _d(_data(c.rec, "int", c.B)))
    return out


# ------------------------------------------------------------------------------------------------------- premises
def _multiple(t, q):
    return bool(((t / q) == (t / q).round()).all())


def _check_int_premises(rec, B):
    d = _data(rec, "int", B)
    x, w, b, om_w, om_b = (d[k].double() for k in ("x", "w", "b", "om_w", "om_b"))
    assert set(x.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert set(w.unique().tolist()) <= {-1.0, 0.0, 1.0}
    assert int((w.reshape(w.shape[0], -1) != 0).sum(1).max()) <= INT_NNZ
    assert _multiple(b, 1) and b.abs().max() <= 4
    # offsets: multiples of 1/4, |w| <= 4 (bf16-exact; fp16x2 pre-scales max|w| into [2^12, 2^13) < 65504)
    assert _multiple(om_w[:18], 0.25) and om_w[:18].abs().max() <= 4 and _multiple(om_b[:18], 0.25)
    # masks: zero rows, logits 0 / +-200, neighbouring taps differ
    assert bool((om_w[18:] == 0).all())
    logits = om_b[18:].tolist()
    assert set(logits) <= set(MASK_LOGIT) and all(logits[t] != logits[t + 1] for t in range(8))
    ph, pw, _, _, _ = _field(x, om_w, om_b)
    assert _multiple(ph, 0.25) and _multiple(pw, 0.25) and max(ph.abs().max(), pw.abs().max()) < 2 ** 20
    col = _columns(x, om_w, om_b)
    col = torch.where(col.abs() < 1e-30, torch.zeros_like(col), col)     # sigmoid(-200): 1e-87, rounded away
    assert _multiple(col, 1 / 32) and col.abs().max() <= 1
    y = _dcn64({"x": x, "w": w, "b": b, "om_w": om_w, "om_b": om_b}).float().double()
    assert _multiple(y, 1 / 32) and y.abs().max() < 2 ** 10


@pytest.mark.parametrize("idx", [i for i, _ in DCN], ids=_ids(DCN))
def test_dcn_int_premises(idx):
    _check_int_premises(CASES[idx].rec, CASES[idx].B)


@pytest.mark.parametrize("rec", _census_dcn(), ids=lambda r: r.label())
def test_dcn_int_premises_of_the_backbones(rec):
    _check_int_premises(rec, 2)


@pytest.mark.parametrize("idx", [i for i, _ in DCN], ids=_ids(DCN))
def test_dcn_coord_positions_are_exact(idx):
    c = CASES[idx]
    for variant in ("coord", "coord-bf16"):
        d = _d(_data(c.rec, variant, c.B))
        x, om_w, om_b = d["x"], d["om_w"], d["om_b"]
        assert _multiple(x[:, :COORD_CH], 1) and x[:, :COORD_CH].abs().max() <= 8
        assert bool((om_w[:18, COORD_CH:] == 0).all()) and _multiple(om_w[:18], 0.25) and _multiple(om_b[:18], 0.25)
        ph, pw, _, _, _ = _field(x, om_w, om_b)
        assert _multiple(ph, 0.25) and _multiple(pw, 0.25)
        assert ph.std() > 0.5 and pw.std() > 0.5                         # positions vary over space
        assert x[:, COORD_CH:].std() > 0.5                               # the sampled values are real
        if variant == "coord-bf16":
            assert bool((x == x.float().bfloat16().double()).all())


# ----------------------------------------------------------------------------------------------------------- reach
@pytest.mark.parametrize("idx", [i for i, c in DCN if c.claims], ids=_ids([(i, c) for i, c in DCN if c.claims]))
def test_dcn_case_reaches_what_it_claims(idx, reached):
    case = CASES[idx]
    assert case.claims <= set(DCN_CLAIMS), case.claims
    got, pairs = reached[idx]
    missing = sorted(case.claims - got)
    assert not missing, f"{case.label()}: claims {missing} it does not reach; class pairs missing: " \
                        f"{sorted(set((h, w) for h in range(6) for w in range(6)) - pairs)}"


def test_dcn_cases_reach_every_class_pair_on_every_family(reached):
    want = {(h, w) for h in range(6) for w in range(6)}
    per = {}
    for i, c in DCN:
        for pkey, ks in c.routes.items():
            for k in ks:
                f = _family(pkey, k)
                if f:
                    per.setdefault(f, set()).update(reached[i][1])
    assert set(per) == {"tensor-core P = 1", "tensor-core P = 2", "CUDA-core", "split fp32 island"}, sorted(per)
    for f, pairs in per.items():
        missing = sorted(want - pairs)
        assert not missing, f"{f}: no case samples the class pairs " + \
            ", ".join(f"({DCN_CLASSES_H[h]}, {DCN_CLASSES_H[w]})" for h, w in missing)
    tags = set().union(*(reached[i][0] for i, c in DCN if c.claims))
    assert tags == set(DCN_CLAIMS), sorted(set(DCN_CLAIMS) - tags)


def test_constructed_dcn_cases_launch_every_dcn_kernel():
    dcn_kernels = {k for k in ROUTES if _family("", k)}
    assert not dcn_kernels & set(UNREACHABLE)
    launched = set()
    for _, c in DCN:
        if c.claims:
            for ks in c.routes.values():
                launched |= {k for k in ks if _family("", k)}
    assert launched == dcn_kernels, sorted(dcn_kernels - launched)


# ---------------------------------------------------------------------------------------------------- discrimination
@pytest.mark.parametrize("idx", [i for i, _ in DCN], ids=_ids(DCN))
def test_dcn_data_discriminates(idx):
    """the float64 reference (oracle.dcn_ref through tests/layer_census.py) equals the restatement here, and each bug
    changes it; "every sample from image 0" needs B >= 2"""
    case = CASES[idx]
    data = _data(case.rec, "int", case.B)
    d = _d(data)
    ref = _reference(case.rec, data)
    assert torch.allclose(ref, _dcn64(d), rtol=0, atol=1e-12)
    same = [bug for bug in BUGS if (case.B >= 2 or bug != "every sample from image 0") and
            torch.equal(_dcn64(d, bug=bug).float(), ref.float())]
    assert not same, f"{case.label()}: the data does not tell the reference from: {same}"


@pytest.mark.parametrize("idx", [i for i, c in DCN if c.rec.arg("x")[2] * c.rec.arg("x")[3] <= 160],
                         ids=_ids([(i, c) for i, c in DCN if c.rec.arg("x")[2] * c.rec.arg("x")[3] <= 160]))
def test_dcn_reference_matches_the_literal_loops(idx):
    """oracle.dcn_ref.dcn_v2_forward against dcn_v2_forward_loops on the case's sampling field (four channels: the
    positions do not depend on the channel count)"""
    from oracle import dcn_ref
    case = CASES[idx]
    d = _d(_data(case.rec, "int", case.B))
    x = d["x"]
    _, _, mask, dh, dw = _field(x, d["om_w"], d["om_b"])
    off = torch.stack([dh, dw], 2).reshape(x.shape[0], 18, x.shape[2], x.shape[3])
    xs, ws = x[:, :4], d["w"][:8, :4]
    vec = dcn_ref.dcn_v2_forward(xs, ws, d["b"][:8], off, mask)
    lit = torch.from_numpy(dcn_ref.dcn_v2_forward_loops(xs.numpy(), ws.numpy(), d["b"][:8].numpy(), off.numpy(),
                                                        mask.numpy()))
    assert torch.allclose(vec, lit, rtol=0, atol=1e-12)
    ph, pw, _, _, _ = _field(x, d["om_w"], d["om_b"])
    H, W = x.shape[2], x.shape[3]
    for p, S in ((ph, H), (pw, W)):
        assert all(bool((p == v).any()) for v in (-1, S - 1, S)), "the field misses exactly -1, S-1 or S"


# ------------------------------------------------------------------------------------------- 32-bit gather offsets
@pytest.mark.parametrize("precision,C,expect", [("bf16", 64, None), ("bf16", 256, "2^31 elements"),
                                                ("bf16x2", 64, None), ("bf16x2", 128, "4 GiB"),
                                                ("fp16x2", 256, "4 GiB")])
def test_dcn_gather_offsets_refused_before_they_overflow(precision, C, expect):
    """A hand-built tensor-core DCN op of B x H x W x C = 2 x 2048 x 2048 x C elements (2^31 at C = 256, 2^30 at
    C = 128): the library refuses it at prepare time when its 32-bit gather offsets would overflow, and launches
    nothing.  The addresses are never dereferenced: the refusal comes first, and a shape it accepts stops at the
    tensor-map encoding, which needs the device (so only the refusals are asserted on a machine without one)."""
    from centerpose_b200 import _lib
    from centerpose_b200 import plan as P
    if not os.path.exists(_lib.LIBPATH):
        pytest.skip("the CUDA library has not been built")
    L = _lib.lib()
    op = P.OpStruct()
    op.type, op.flags, op.act_dtype = P.OP_DCN, P.FLAG_TC | P.FLAG_RELU, P.PRECISIONS[precision]
    op.B, op.H, op.W, op.Ho, op.Wo, op.nsrc, op.cout = 2, 2048, 2048, 2048, 2048, 1, 64
    op.cin[0] = C
    op.kh = op.kw = 3
    op.stride, op.pad_h, op.pad_w = 1, 1, 1
    op.Hd, op.Wd, op.out_sy, op.out_sx = 2048, 2048, 1, 1
    op.src[0] = op.aux = op.dst = op.weight = op.bias = 1 << 20          # never dereferenced
    op.aux_pitch = 32
    op.acc_scale = 1.0
    ops = (P.OpStruct * 1)(op)
    before = L.cpb200_launch_count()
    rc = L.cpb200_prepare_ops(ops, 1)
    err = L.cpb200_last_error().decode()
    L.cpb200_release_ops(ops, 1)
    assert L.cpb200_launch_count() == before
    if expect is not None:
        assert rc != 0 and expect in err, (rc, err)
    else:
        assert rc == 0 or "32-bit gather offsets" not in err, err
