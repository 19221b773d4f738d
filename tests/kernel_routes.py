"""Route table and edge-case list of the network ops (tests/test_kernel_envelope_gpu.py, tests/test_kernel_routes_cpu.py).
A helper module: it holds no tests.

``ROUTES`` names every kernel instantiation the op dispatcher can launch for a network op, as the normalised key
``kernel_key`` makes of its demangled name (``conv_tc_kernel<64,false,2>``, ``maxpool_kernel<SpC,SpM>``), with the
predicate or branch that selects it.  ``CASES`` are ``Record`` s built by hand (not recorded from a model) at both sides of
the boundaries of those predicates and of the prepare functions; each declares, per precision, the exact set of kernels
its program launches, and why it exists.

Precision keys of ``Case.routes``: "fp32", "bf16", "bf16x2", "fp16x2", "x2" (both split precisions: they launch the same
kernels) and "bf16-simt" (bf16 with PlanBuilder(tc=False): the CUDA-core kernels).
"""
from __future__ import annotations

import inspect
import re
from dataclasses import dataclass, field
from typing import Dict, FrozenSet, Optional, Tuple

from tests.layer_census import Record

CVT_IN, CVT_OUT = "convert_from_split_kernel", "convert_to_split_kernel"
S2D = "s2d_split_kernel"


def kernel_key(name: str) -> str:
    """normalised kernel name: namespaces, casts, 'const', whitespace and the parameter list dropped, bool template
    arguments spelled false / true.  Takes cu++filt's demangling and the library route log's (__cxa_demangle) alike."""
    s = name.strip()
    s = re.sub(r"^void\s+", "", s)
    s = s.replace("(anonymous namespace)::", "").replace("<unnamed>::", "").replace("cpb::", "")
    s = s.replace("(bool)0", "false").replace("(bool)1", "true").replace("(int)", "")
    depth, cut = 0, len(s)
    for i, ch in enumerate(s):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    s = s[:cut]
    s = re.sub(r"\bconst\b", "", s).replace("__nv_bfloat16", "bf16")
    return re.sub(r"\s+", "", s)


# ------------------------------------------------------------------------------------------------------ kernel keys
def k_tc(bn, p, dcn=False):
    return f"conv_tc_kernel<{bn},{'true' if dcn else 'false'},{p}>"


def k_c3(bn, p):
    return f"conv3x3_tc_kernel<{bn},{p}>"


def k_sp(c, n, s, p):
    return f"conv_sp_kernel<{c},{n},{s},{p}>"


def k_simt(t, cout, dcn=False):
    m, n = (256, 16) if cout <= 16 else (128, 32) if cout <= 32 else (64, 64)
    return f"conv_simt_kernel<{t},{m},{n},{'true' if dcn else 'false'}>"


def k_stem(t, co, px, st, kw):
    return f"stem_kernel<{t},{co},{px},{st},{kw}>"


FMT = {"fp32": ("float*", "float*"), "bf16": ("bf16*", "bf16*"), "x2": ("SpC", "SpM")}


def k_elt(name, fmt, vec=None):
    pi, po = FMT[fmt]
    return f"{name}<{'' if vec is None else str(vec) + ','}{pi},{po}>"


# ------------------------------------------------------------------------------------------------------ route table
def _routes():
    r = {}
    tc = "net.cu route TAP: net_tc.cu tap_prepare (not c3_eligible / sp_eligible; PlanBuilder._tc_ok: Wo >= 8); BN = tc::bn_for: " \
         "next pow2 >= cout, <= 256, split <= 128; tap_run switch"
    for bn in (16, 32, 64, 128):
        for p in (1, 2):
            r[k_tc(bn, p)] = tc
    r[k_tc(256, 1)] = tc
    dcn = "net.cu route TAP: net_tc.cu tap_prepare DCN branch (PlanBuilder.dcn: C % 64 == 0, cout % 16 == 0, cout >= 32, W >= 8); " \
          "BN <= 128 / P"
    for bn, p in ((32, 1), (64, 1), (128, 1), (32, 2), (64, 2)):
        r[k_tc(bn, p, True)] = dcn
    c3 = "net.cu route HALO: net_tc3.cu c3_eligible (3x3 / 5x5 / 7x1 / 1x7, stride 1, same padding, one dense input, Ho, Wo >= 8) + c3_run switch"
    for bn in (16, 32, 64, 128):
        for p in (1, 2):
            r[k_c3(bn, p)] = c3
    r[k_c3(256, 1)] = c3
    for c in (16, 32):
        for n in (16, 32, 64):
            for s in (1, 2):
                for p in (1, 2):
                    r[k_sp(c, n, s, p)] = "net.cu route SP: net_tc_sp.cu sp_eligible (3x3 pad 1, cin 16 / 32, cout 16 / 32 / 64, Wo >= 8) + dispatch_n"
    for n in (16, 64):
        r[f"stem_tc_kernel<{n},2>"] = "net.cu route STEM: net_stem_tc.cu stem_tc_eligible + stem_tc_run (bf16, stride 2)"
        for p in (1, 2):
            r[f"stem_tc_h_kernel<{n},{p}>"] = "net.cu route STEM: net_stem_tc.cu stem_tc_eligible + stem_tc_run (stride 1)"
    for p in (1, 2):
        r[f"heads_tc_kernel<{p}>"] = "net.cu route HEADS: net_heads.cu heads_prepare / heads_run (plan.py Plan._fuse_heads)"
    for t in ("float", "bf16"):
        for co in (16, 32, 64):
            for d in (False, True):
                r[k_simt(t, co, d)] = "net_simt.cu launch_conv (cout <= 16 / <= 32 / more)"
        for co, px, st, kw in ((64, 1, 2, 3), (16, 4, 2, 3), (16, 4, 1, 7), (16, 4, 2, 7), (32, 2, 2, 7), (64, 1, 2, 7),
                               (64, 1, 1, 7)):
            r[k_stem(t, co, px, st, kw)] = "net_simt.cu run_op_simt STEM switch"
    for fmt in ("fp32", "bf16", "x2"):
        vec, fast = (4, 4) if fmt == "fp32" else (8, 8) if fmt == "bf16" else (4, 8)
        r[k_elt("maxpool_kernel", fmt)] = "net_simt.cu run_eltwise MAXPOOL"
        r[k_elt("dwdeconv_add_fast_kernel", fmt, fast)] = "net_simt.cu run_eltwise DWDECONV_ADD: f, C / VEC pow2, (256 / CV) % f == 0"
        r[k_elt("dwdeconv_add_kernel", fmt, vec)] = "net_simt.cu run_eltwise DWDECONV_ADD: generic"
        r[k_elt("dwconv_kernel", fmt, vec)] = "net_simt.cu run_eltwise DWCONV: generic (k = 7)"
        for kk, ss, px in ((3, 1, 4), (5, 1, 4), (3, 2, 2), (5, 2, 2)):
            pi, po = FMT[fmt]
            r[f"dwconv_tiled_kernel<{vec},{kk},{ss},{px},{pi},{po}>"] = "net_simt.cu run_eltwise DWCONV: DW_TILED"
        pi, po = FMT[fmt]
        r[f"avgpool_kernel<{pi},{'float*' if fmt == 'x2' else po}>"] = "net_simt.cu run_eltwise AVGPOOL"
        r[f"scale_add_kernel<{pi},{'float*' if fmt == 'x2' else po},{po}>"] = "net_simt.cu run_eltwise SCALE_ADD"
        r[k_elt("upsample_add_kernel", fmt)] = "net_simt.cu run_eltwise UPSAMPLE_ADD"
        r[k_elt("avgpool2_kernel", fmt)] = "net_simt.cu run_eltwise AVGPOOL2"
        r[k_elt("resize_bilinear_kernel", fmt)] = "net_simt.cu run_eltwise RESIZE_BILINEAR"
    r[CVT_IN] = "net_simt.cu run_op_split CONVERT (FLAG_TO_F32): entry of an fp32 island"
    r[CVT_OUT] = "net_simt.cu run_op_split CONVERT: exit of an fp32 island"
    r[S2D] = "net_simt.cu run_op_split S2D (PlanBuilder.stem: split, stride 2, even H, W)"
    return r


ROUTES: Dict[str, str] = _routes()

# instantiations no PlanBuilder call can reach, with the reason (tests/test_kernel_routes_cpu.py checks the lists against
# the library's kernels)
UNREACHABLE = {
    k_tc(16, 1, True): "PlanBuilder.dcn sends cout < 32 to the CUDA-core kernel, so the DCN tile is never 16 wide",
    k_tc(16, 2, True): "PlanBuilder.dcn sends cout < 32 to the CUDA-core kernel, so the DCN tile is never 16 wide",
}


# ------------------------------------------------------------------------------------------------------------- cases
def sym(C, H, W, kind="act", pc=0, off=0):
    return ("sym", C, H, W, kind, pc, off)


def tensor(*shape):
    return ("tensor", tuple(shape))


def record(method, **kw) -> Record:
    """a Record of PlanBuilder.<method>(**kw) (descriptors as arguments), defaults applied as the census records them"""
    from centerpose_b200.plan import PlanBuilder
    sig = inspect.signature(getattr(PlanBuilder, method))
    bound = sig.bind(None, **kw)
    bound.apply_defaults()
    return Record(method, tuple((k, v) for k, v in bound.arguments.items() if k != "self"), ())


@dataclass(frozen=True)
class Case:
    rec: Record
    routes: Dict[str, FrozenSet[str]]          # precision key -> kernels the program launches
    reason: str
    B: int = 1
    error: Optional[str] = None                # an expected CPB200_ERR_ARG: a fragment of its message
    randn_only: bool = False                   # no integer-exact leg (hswish / hsigmoid, pools over 2^k-free sizes)
    claims: FrozenSet[str] = frozenset()       # DCN: what its "int" data reaches (tests/test_dcn_cases_cpu.py)

    def precisions(self):
        out = []
        for k in self.routes:
            out += ["bf16x2", "fp16x2"] if k == "x2" else [k]
        return out

    def routes_for(self, precision):
        key = "x2" if precision in ("bf16x2", "fp16x2") and "x2" in self.routes else precision
        return self.routes[key]

    @property
    def exact(self):
        from tests.replay import INT_EXACT
        act = dict(self.rec.args).get("act")
        return not self.randn_only and self.rec.method in INT_EXACT and act not in ("hswish", "hsigmoid")

    def label(self):
        return f"{self.rec.label()} B={self.B}: {self.reason}"


def _fs(*ks):
    return frozenset(ks)


CASES = []


def add(method, routes, reason, B=1, error=None, randn_only=False, claims=(), **kw):
    CASES.append(Case(record(method, **kw), {k: frozenset(v) for k, v in routes.items()}, reason, B, error, randn_only,
                      frozenset(claims)))


def island(*ks):
    """the kernels of an fp32 island in the split precisions"""
    return {CVT_IN, *ks, CVT_OUT}


def conv(cin, cout, H, W, k=3, stride=1, pad=None, routes=None, reason="", B=1, srcs=None, out="act", res=False, act=None,
         relu=False, kwh=None):
    """one conv case (kwh = (kh, kw): a non-square filter with same padding); fp32 (CUDA-core) joins every case whose
    routes do not name it.  An NCHW output is written at channel offset 2 of a destination with two spare channels on
    each side (tests/replay.py)."""
    kh, kw = kwh or (k, k)
    pad_hw = (kh // 2, kw // 2) if kwh else None
    ph, pw = pad_hw or ((kh // 2, kw // 2) if pad is None else (pad, pad))
    srcs = srcs or (sym(cin, H, W),)
    cin = sum(s[1] for s in srcs)
    Ho = (H + 2 * ph - kh) // stride + 1
    Wo = (W + 2 * pw - kw) // stride + 1
    routes = dict(routes)
    routes.setdefault("fp32", {k_simt("float", cout)})
    extra = dict(dst=sym(cout, Ho, Wo, "nchw_out")) if out == "nchw" else {}
    add("conv", routes, reason, B=B, srcs=tuple(srcs), w=tensor(cout, cin, kh, kw), b=tensor(cout), stride=stride,
        pad=0 if pad_hw else ph, pad_hw=pad_hw, relu=relu, res=sym(cout, Ho, Wo) if res else None, out=out, act=act,
        **extra)


def tcr(bn1, bn2, **more):
    """routes of a conv on the tap-per-stage kernel: bf16 tile bn1, split tile bn2"""
    return {"bf16": {k_tc(bn1, 1)}, "x2": {k_tc(bn2, 2)}, **more}


def c3r(bn1, bn2, **more):
    return {"bf16": {k_c3(bn1, 1)}, "x2": {k_c3(bn2, 2)}, **more}


# ---- conv_tc_kernel (net_tc.cu): 1x1, stride 2, multi-input, slices, NCHW / f32 outputs, Ho < 8 ----
conv(64, 16, 12, 20, k=1, routes=tcr(16, 16), reason="1x1, BN 16, TW 16 x TH 8 (Wo >= 16), partial tile rows")
conv(96, 32, 9, 9, k=1, routes=tcr(32, 32), reason="cin 96 (bk 32), BN 32, Wo = 9: TW 8 + 1 column")
conv(64, 48, 17, 23, stride=2, routes=tcr(64, 64), reason="3x3 stride 2, odd H and W, cout 48 partial 64 tile")
conv(64, 48, 17, 23, stride=2, pad=0, routes=tcr(64, 64), reason="3x3 stride 2 pad 0 (k > 1)")
conv(48, 112, 8, 16, k=1, routes=tcr(128, 128), reason="cin 48 (bk 16), BN 128 partial (112), Wo = 16 exactly")
conv(512, 144, 8, 8, k=1, routes=tcr(256, 128),
     reason="cin 512 (8 K slabs); bf16 BN 256 partial; split BN 128 n_tiles 2 with a partial last tile")
conv(64, 384, 9, 17, k=1, routes=tcr(256, 128), reason="BN 256 n_tiles 2, partial last N tile (384 = 256 + 128)")
conv(64, 64, 7, 11, routes=tcr(64, 64),
     reason="3x3 with Ho < 8 <= Wo (a 224x352 input's 1/32 map): not c3_eligible, one tile row of TH 16 holds 7 valid rows")
conv(64, 64, 4, 8, routes=tcr(64, 64), B=3, reason="Ho 4, Wo = 8 exactly: smallest map the tap-per-stage kernel takes")
conv(64, 64, 11, 7, routes={"bf16": {k_simt("bf16", 64)}, "x2": island(k_simt("float", 64))},
     reason="Wo < 8 <= Ho: no tensor-core kernel, an fp32 island in the split precisions")
conv(0, 32, 10, 16, srcs=(sym(16, 10, 16), sym(64, 10, 16), sym(32, 10, 16), sym(48, 10, 16)), routes=tcr(32, 32),
     reason="four inputs of mixed width 16 + 64 + 32 + 48: bk 16 over all four tensor maps")
conv(0, 64, 9, 9, k=1, srcs=(sym(32, 9, 9), sym(64, 9, 9)), routes=tcr(64, 64), res=True, relu=True,
     reason="two inputs 32 + 64 (bk 32), relu + residual")
conv(0, 32, 9, 12, k=1, srcs=(sym(32, 9, 12, pc=96, off=32),), routes=tcr(32, 32),
     reason="channel-slice input at offset 32 of 96 (src_pitch), every format")
conv(0, 48, 8, 10, srcs=(sym(16, 8, 10, pc=64, off=0),), routes=tcr(64, 64),
     reason="3x3 on a channel slice at offset 0 of 64: not c3 / sp (src_pitch), tap-per-stage kernel")
conv(0, 16, 9, 9, k=1, srcs=(sym(64, 9, 9, pc=128, off=64), sym(32, 9, 9)), routes=tcr(16, 16),
     reason="slice at offset 64 beside a dense input")
conv(64, 5, 9, 13, k=1, out="nchw", routes=tcr(16, 16), reason="cout 5, NCHW fp32 output")
conv(96, 27, 8, 9, out="nchw", routes=tcr(32, 32), reason="cout 27, 3x3 NCHW output")
conv(64, 1, 10, 8, k=1, out="nchw", routes=tcr(16, 16), reason="cout 1, NCHW")
conv(64, 27, 9, 11, k=1, out="f32", routes=tcr(32, 32), reason="cout 27, NHWC fp32 output")
conv(64, 48, 9, 16, k=1, out="nchw", routes=tcr(64, 64), reason="cout 48 NCHW, TW 16")
conv(64, 64, 96, 128, k=1, B=3, routes=tcr(64, 64), reason="288 tiles > 2 x 132 SMs: the persistent loop wraps twice")
conv(64, 64, 9, 17, k=1, res=True, act="hswish", routes=tcr(64, 64), reason="hswish + residual epilogue")
conv(64, 64, 9, 17, k=1, res=True, act="hsigmoid", routes=tcr(64, 64), reason="hsigmoid + residual epilogue")
conv(64, 64, 9, 17, k=1, act="hswish", routes=tcr(64, 64), reason="hswish, no residual")
conv(64, 64, 9, 17, k=1, act="hsigmoid", routes=tcr(64, 64), reason="hsigmoid, no residual")

# ---- conv3x3_tc_kernel (net_tc3.cu): ring regimes from c3_prepare's arithmetic ----
conv(64, 16, 16, 8, routes=c3r(16, 16), reason="Ho = TH, Wo = TW: one tile; bk 64: resident, na 3 (P1) / 4 (P2)")
conv(48, 32, 17, 9, routes=c3r(32, 32), reason="TH + 1, TW + 1: partial tiles both ways; bk 16: resident, na 16")
conv(96, 48, 15, 8, routes=c3r(64, 64), res=True, relu=True,
     reason="TH - 1; bk 32: P1 resident na 8, P2 streamed na 8 nb 8; relu + residual")
conv(64, 128, 8, 9, B=3, routes=c3r(128, 128), reason="Ho = 8; P1 resident na 3, P2 streamed na 4 nb 4")
conv(64, 256, 9, 8, routes=c3r(256, 128), reason="cout 256: P1 BN 256 streamed na 3 nb 4; P2 BN 128 x 2 streamed")
conv(64, 384, 17, 15, routes=c3r(256, 128), reason="cout 384: P1 BN 256 x 2 (partial last), P2 BN 128 x 3; streamed")
conv(512, 64, 9, 9, routes=c3r(64, 64), reason="cin 512: weights streamed (na 3 / 4, nb 8)")
conv(16, 128, 33, 17, routes=c3r(128, 128), reason="cin 16: bk 16 halo, resident na 16; three tile rows")
conv(32, 128, 16, 16, routes=c3r(128, 128), reason="cin 32: resident, na 8 (P1) / 6 (P2 reduced to fit)")
conv(16, 64, 9, 11, k=5, routes=c3r(64, 64), reason="5x5 bk 16: resident na 8")
conv(64, 64, 8, 8, k=5, routes=c3r(64, 64), reason="5x5 bk 64: streamed na 3 nb 8 (P1) / na 4 nb 6 (P2)")
conv(64, 64, 9, 8, kwh=(7, 1), routes=c3r(64, 64), reason="7x1: resident na 3 (P1) / 4 (P2)")
conv(32, 64, 17, 9, kwh=(7, 1), routes=c3r(64, 64), reason="7x1 bk 32: resident na 8")
conv(64, 64, 8, 17, kwh=(1, 7), routes=c3r(64, 64), reason="1x7: resident na 3")
conv(128, 64, 9, 9, kwh=(1, 7), routes=c3r(64, 64), reason="1x7 cin 128: P1 resident na 3, P2 streamed na 4 nb 6")
conv(64, 32, 16, 8, res=True, act="hswish", routes=c3r(32, 32), reason="halo kernel, hswish + residual")
conv(64, 32, 16, 8, res=True, act="hsigmoid", routes=c3r(32, 32), reason="halo kernel, hsigmoid + residual")
conv(64, 64, 96, 128, B=3, routes=c3r(64, 64), reason="288 halo tiles (6 x 16 x 3) > 2 x 132 SMs: the persistent loop wraps")
conv(64, 27, 9, 9, out="f32", routes=c3r(32, 32), reason="halo kernel, cout 27 fp32 output (c3 takes OUT_F32)")

# ---- conv_sp_kernel (net_tc_sp.cu): every (C, N, S) ----
_SP_SIZES = [(8, 8), (9, 9), (16, 8), (17, 9), (15, 23), (33, 17)]
for i, (c, n, s) in enumerate((c, n, s) for c in (16, 32) for n in (16, 32, 64) for s in (1, 2)):
    H, W = _SP_SIZES[i % len(_SP_SIZES)]
    if s == 2:
        H, W = 2 * H - 1, 2 * W - 1                         # odd sizes: Ho = H, Wo = W of the table
    conv(c, n, H, W, stride=s, routes={"bf16": {k_sp(c, n, s, 1)}, "x2": {k_sp(c, n, s, 2)}},
         res=(i % 3 == 0), relu=(i % 2 == 0), reason=f"small-channel kernel C {c} N {n} stride {s}")

# ---- CUDA-core conv (fp32, bf16 with tc=False) ----
for co in (16, 27, 48):
    conv(32, co, 9, 7, routes={"bf16-simt": {k_simt("bf16", co)}}, out="nchw" if co % 16 else "act",
         reason=f"CUDA-core conv, cout {co} (tile {k_simt('float', co)})")

# ---- DCN ----
# Every DCN case runs three legs: dyadic data (exact sampling positions, exact result), "coord" data (exact positions,
# real-valued samples, conv bounds) and randn data.  ``claims`` name what a case's dyadic data reaches, as
# tests/test_dcn_cases_cpu.py computes it from the data in float64:
#   "all-pairs"   every (h-class, w-class) pair of sampling classes (DCN_CLASSES) on a tap whose mask is not 0
#   "beyond-tile" samples inside the map displaced by more than the tensor-core tile: one with |dh| > TH, one with
#                 |dw| > TW
#   "beyond-map"  a displacement larger than the map: |dh| > H or |dw| > W
#   "masks"       each mask value (0, 0.5, 1) on at least two taps
#   "last-pixel"  B >= 2 and a sample of the last image that reads its last row and column with a nonzero weight
DCN_CLASSES = ("p <= -1", "-1 < p < 0", "integer p in [0, S-1]", "fractional p in (0, S-1)", "S-1 < p < S", "p >= S")
DCN_CLAIMS = ("all-pairs", "beyond-tile", "beyond-map", "masks", "last-pixel")


def dcn(cin, cout, H, W, routes, reason, B=1, claims=()):
    add("dcn", routes, reason, B=B, claims=claims, x=sym(cin, H, W), w=tensor(cout, cin, 3, 3), b=tensor(cout),
        om_w=tensor(27, cin, 3, 3), om_b=tensor(27))


def _dcn_simt(t, cin, cout):
    return {k_simt(t, 32), k_simt(t, cout, True)}


dcn(64, 32, 9, 8, {"fp32": _dcn_simt("float", 64, 32), "bf16": {k_c3(32, 1), k_tc(32, 1, True)},
                   "x2": {k_c3(32, 2), k_tc(32, 2, True)}}, reason="DCN cout 32, W = 8")
dcn(128, 48, 8, 12, {"fp32": _dcn_simt("float", 128, 48), "bf16": {k_c3(32, 1), k_tc(64, 1, True)},
                     "x2": {k_c3(32, 2), k_tc(64, 2, True)}}, reason="DCN cin 128, cout 48 (partial 64 tile)", B=3)
dcn(64, 256, 17, 9, {"bf16": {k_c3(32, 1), k_tc(128, 1, True)}, "x2": {k_c3(32, 2), k_tc(64, 2, True)}},
    reason="DCN cout 256: BN 128 x 2 (bf16) / 64 x 4 (split)")
dcn(64, 64, 5, 12, {"bf16": {k_tc(32, 1), k_tc(64, 1, True)}, "x2": {k_tc(32, 2), k_tc(64, 2, True)}},
    reason="DCN H < 8 <= W: offset conv on the tap-per-stage kernel")
dcn(64, 64, 12, 6, {"bf16": {k_simt("bf16", 32), k_simt("bf16", 64, True)},
                    "x2": island(k_simt("float", 32), k_simt("float", 64, True))},
    reason="DCN W < 8: CUDA-core offset conv and DCN (fp32 island in the split precisions)")
dcn(64, 16, 9, 9, {"bf16-simt": {k_simt("bf16", 32), k_simt("bf16", 16, True)}, "fp32": _dcn_simt("float", 64, 16)},
    reason="DCN cout 16 on the CUDA-core kernel (bf16 with tc=False)")
dcn(64, 32, 9, 9, {"bf16-simt": {k_simt("bf16", 32), k_simt("bf16", 32, True)}}, reason="bf16 CUDA-core DCN, cout 32")
dcn(64, 64, 9, 9, {"bf16-simt": {k_simt("bf16", 32), k_simt("bf16", 64, True)}}, reason="bf16 CUDA-core DCN, cout 64")


# ---- stems ----
def stem(co, k, stride, H, W, routes, reason, B=1, error=None, act=None):
    add("stem", routes, reason, B=B, error=error, randn_only=act is not None, x=sym(3, H, W, "nchw_in"),
        w=tensor(co, 3, k, k), b=tensor(co), k=k, stride=stride, pad=k // 2, act=act)


for t, pk in (("float", "fp32"), ("bf16", "bf16-simt")):
    for co, px, st, kw in ((64, 1, 2, 3), (16, 4, 2, 3), (16, 4, 1, 7), (16, 4, 2, 7), (32, 2, 2, 7), (64, 1, 2, 7),
                           (64, 1, 1, 7)):
        # Wo % PX == 0: a multiple of 4 (and of PX) columns; odd heights
        W = 16 * st if px > 1 else 13 * st + (st - 1)
        stem(co, kw, st, 9 * st + 1, W, {pk: {k_stem(t, co, px, st, kw)}}, f"CUDA-core stem CO {co} PX {px} stride {st} {kw}x{kw}")
        if px > 1:
            stem(co, kw, st, 9, 17, {pk: set()}, f"CUDA-core stem PX {px}: an odd Wo (Wo % PX != 0) is refused",
                 error="not a multiple of")
stem(16, 7, 1, 17, 23, {"bf16": {"stem_tc_h_kernel<16,1>"}, "x2": {"stem_tc_h_kernel<16,2>"}},
     reason="tensor-core stem, stride 1, co 16, odd sizes")
stem(64, 7, 1, 9, 13, {"bf16": {"stem_tc_h_kernel<64,1>"}, "x2": {"stem_tc_h_kernel<64,2>"}}, B=3,
     reason="tensor-core stem, stride 1, co 64")
stem(16, 7, 2, 33, 47, {"bf16": {"stem_tc_kernel<16,2>"}, "x2": {k_stem("float", 16, 4, 2, 7), CVT_OUT}},
     reason="stride 2, odd sizes: bf16 im2col stem; split: fp32 stem (odd H / W have no space-to-depth)")
stem(64, 7, 2, 34, 30, {"bf16": {"stem_tc_kernel<64,2>"}, "x2": {S2D, k_c3(64, 2)}},
     reason="stride 2, even sizes: split space-to-depth + 5x5 halo conv on the 17x15 half map")
stem(64, 3, 2, 34, 18, {"x2": {S2D, k_sp(16, 64, 1, 2)}, "fp32": {k_stem("float", 64, 1, 2, 3)}},
     reason="3x3 stride-2 stem: space-to-depth + 3x3 small-channel conv (HRNet)")
stem(16, 3, 2, 32, 48, {"x2": {S2D, k_sp(16, 16, 1, 2)}, "bf16": {k_stem("bf16", 16, 4, 2, 3)}}, act="hswish",
     reason="MobileNetV3 stem: 3x3 stride 2, hswish")

# ---- element-wise ops: every format ----
ELT = ("fp32", "bf16", "x2")


def elt(method, kernels, reason, randn_only=False, B=1, **kw):
    """kernels(format) -> the kernel key, or the set of keys, the op launches in that activation format"""
    routes = {}
    for f in ELT:
        k = kernels(f)
        routes[f] = {k} if isinstance(k, str) else k
    add(method, routes, reason, B=B, randn_only=randn_only, **kw)


def up_add(C, f, H, W, fast, reason, skip=True):
    k = 2 * f
    Ho = (H - 1) * f - 2 * (f // 2) + k
    Wo = (W - 1) * f - 2 * (f // 2) + k
    vec = {"fp32": 4, "bf16": 8, "x2": 4}
    fvec = {"fp32": 4, "bf16": 8, "x2": 8}
    elt("up_add", lambda fm: k_elt("dwdeconv_add_fast_kernel", fm, fvec[fm]) if fast(fm) else
        k_elt("dwdeconv_add_kernel", fm, vec[fm]), reason, x=sym(C, H, W), skip=sym(C, Ho, Wo) if skip else None,
        w=tensor(C, 1, k, k))


up_add(64, 2, 9, 7, lambda fm: True, "f 2, C / VEC a power of two: fast kernel")
up_add(32, 4, 5, 3, lambda fm: True, "f 4: fast kernel", skip=False)
up_add(48, 3, 5, 7, lambda fm: False, "f 3, C 48: generic kernel")
up_add(80, 3, 4, 5, lambda fm: False, "f 3, C 80: generic kernel", skip=False)
up_add(512, 8, 3, 2, lambda fm: False, "f 8, C 512: (256 / CV) % f != 0 in every format -> generic kernel")
up_add(512, 4, 3, 3, lambda fm: fm != "fp32", "f 4, C 512: fp32 CV 128, (256 / CV) % f != 0 -> generic; "
       "bf16 / split CV 64 -> fast")


def dwconv(C, k, s, H, W, reason, act=None):
    vec = {"fp32": 4, "bf16": 8, "x2": 4}
    px = 4 if s == 1 else 2
    tiled = k in (3, 5)
    elt("dwconv", lambda fm: (f"dwconv_tiled_kernel<{vec[fm]},{k},{s},{px},{FMT[fm][0]},{FMT[fm][1]}>" if tiled
                              else k_elt("dwconv_kernel", fm, vec[fm])), reason, randn_only=act == "hswish",
        x=sym(C, H, W), w=tensor(C, 1, k, k), b=tensor(C), stride=s, act=act)


for k in (3, 5, 7):
    for s in (1, 2):
        dwconv(48 if k == 5 else 32, k, s, 9 + 2 * k, 11 + k, f"dwconv {k}x{k} stride {s}, odd sizes",
               act="relu" if (k + s) % 2 else None)
dwconv(16, 3, 1, 7, 9, "dwconv 3x3 hswish", act="hswish")

elt("maxpool", lambda fm: k_elt("maxpool_kernel", fm), "3x3 / stride 2 / pad 1 on odd sizes", x=sym(32, 17, 23), k=3,
    stride=2, pad=1)
elt("maxpool", lambda fm: k_elt("maxpool_kernel", fm), "3x3 / stride 2 / pad 1, 9x9", x=sym(16, 9, 9), k=3,
    stride=2, pad=1, B=3)
for f, skip, relu in ((2, True, True), (4, False, False), (8, True, False), (4, True, True), (8, False, True)):
    elt("upsample_add", lambda fm: k_elt("upsample_add_kernel", fm), f"nearest upsample x{f}, skip {skip}, relu {relu}",
        x=sym(32, 5, 7), skip=sym(32, 5 * f, 7 * f) if skip else None, f=f, relu=relu)
def avgpool(H, W):
    pow2 = (H * W) & (H * W - 1) == 0                   # a mean over 2^k integers is exact
    elt("avgpool", lambda fm: {f"avgpool_kernel<{FMT[fm][0]},{'float*' if fm == 'x2' else FMT[fm][1]}>"} |
        ({CVT_OUT} if fm == "x2" else set()), f"global average pool over {H}x{W}", randn_only=not pow2, x=sym(64, H, W))


for H, W in ((1, 1), (7, 7), (96, 160)):
    avgpool(H, W)
for skip in (True, False):
    elt("scale_add", lambda fm: {f"scale_add_kernel<{FMT[fm][0]},{'float*' if fm == 'x2' else FMT[fm][1]},{FMT[fm][1]}>"} |
        ({CVT_IN} if fm == "x2" else set()), f"SE gate, skip {skip}", x=sym(48, 9, 11), gate=sym(48, 1, 1),
        skip=sym(48, 9, 11) if skip else None)
elt("avgpool2", lambda fm: k_elt("avgpool2_kernel", fm), "2x2 average pool, odd sizes", x=sym(32, 17, 23))
elt("resize_bilinear", lambda fm: k_elt("resize_bilinear_kernel", fm), "align-corners bilinear 9x11 -> 17x23",
    randn_only=True, x=sym(32, 9, 11), Ho=17, Wo=23)

# ---- cases added after the ones above (appended, so that a case keeps its index in CASES) ----
avgpool(8, 8)
avgpool(16, 32)
elt("resize_bilinear", lambda fm: k_elt("resize_bilinear_kernel", fm),
    "align-corners bilinear 9x11 -> 17x21: ratio 1/2 both ways, exact on integers", x=sym(32, 9, 11), Ho=17, Wo=21)

# constructed sampling: every class pair, displacements past a tile and past the map, B = 2 (the rowb = n * H base)
_ALL = ("all-pairs", "masks", "last-pixel")
dcn(64, 48, 13, 11, {"fp32": _dcn_simt("float", 64, 48), "bf16": {k_c3(32, 1), k_tc(64, 1, True)},
                     "x2": {k_c3(32, 2), k_tc(64, 2, True)}, "bf16-simt": {k_simt("bf16", 32), k_simt("bf16", 48, True)}},
    B=2, claims=_ALL + ("beyond-map",),
    reason="DCN TW 8 x TH 16, partial tiles both ways (13 x 11), cout 48: partial 64 tile")
dcn(128, 96, 11, 23, {"fp32": _dcn_simt("float", 128, 96), "bf16": {k_c3(32, 1), k_tc(128, 1, True)},
                      "x2": {k_c3(32, 2), k_tc(64, 2, True)}},
    B=2, claims=_ALL + ("beyond-map",),
    reason="DCN TW 16 x TH 8, partial tiles both ways (11 x 23), cin 128 (two K slabs), cout 96: partial 128 tile (bf16), "
           "64 + partial 32 (split)")
dcn(256, 32, 9, 17, {"fp32": _dcn_simt("float", 256, 32), "bf16": {k_c3(32, 1), k_tc(32, 1, True)},
                     "x2": {k_c3(32, 2), k_tc(32, 2, True)}, "bf16-simt": {k_simt("bf16", 32), k_simt("bf16", 32, True)}},
    B=2, claims=_ALL + ("beyond-map",), reason="DCN cin 256 (four K slabs), cout 32, TW 16 with one extra column")
dcn(64, 16, 10, 9, {"fp32": _dcn_simt("float", 64, 16), "bf16": {k_c3(32, 1), k_simt("bf16", 16, True)},
                    "x2": island(k_c3(32, 2), k_simt("float", 16, True))},
    B=2, claims=_ALL + ("beyond-map",),
    reason="DCN cout 16: tensor-core offset conv, CUDA-core DCN (an fp32 island in the split precisions)")
dcn(64, 64, 9, 6, {"fp32": _dcn_simt("float", 64, 64), "bf16": {k_simt("bf16", 32), k_simt("bf16", 64, True)},
                   "x2": island(k_simt("float", 32), k_simt("float", 64, True))},
    B=2, claims=_ALL + ("beyond-map",), reason="DCN W = 6 < 8: the split fp32 island, every class pair")
dcn(64, 128, 96, 128, {"bf16": {k_c3(32, 1), k_tc(128, 1, True)}, "x2": {k_c3(32, 2), k_tc(64, 2, True)}},
    B=3, claims=_ALL + ("beyond-tile",),
    reason="DCN 288 tiles (bf16) / 576 (split) > 2 x 132 SMs: the persistent loop wraps and the next unit's corner "
           "loads cross a tile boundary")


# ---- fused heads (Plan._fuse_heads -> heads_tc_kernel): n x (3x3 + ReLU -> 1x1 NCHW) over one input ----
@dataclass(frozen=True)
class HeadCase:
    couts: Tuple[int, ...]
    hid: int
    C: int
    H: int
    W: int
    B: int
    routes: Dict[str, FrozenSet[str]]
    reason: str

    @property
    def fused(self):
        return min(len(self.couts), 8)

    def precisions(self):
        return ["bf16", "bf16x2", "fp16x2"]

    def routes_for(self, precision):
        return self.routes["bf16" if precision == "bf16" else "x2"]

    def label(self):
        return f"heads{self.couts} hid {self.hid} C {self.C} {self.H}x{self.W} B={self.B}: {self.reason}"


HEAD_CASES = []


def heads(couts, hid, C, H, W, B, reason):
    routes = {"bf16": {"heads_tc_kernel<1>"}, "x2": {"heads_tc_kernel<2>"}}
    if len(couts) > 8:                                  # the ninth pair stays a 3x3 + 1x1 conv pair
        bn1 = max(16, 1 << (max(couts[8:]) - 1).bit_length())
        routes = {"bf16": routes["bf16"] | {k_c3(min(hid, 256), 1), k_tc(bn1, 1)},
                  "x2": routes["x2"] | {k_c3(128, 2), k_tc(bn1, 2)}}
    HEAD_CASES.append(HeadCase(tuple(couts), hid, C, H, W, B, {k: frozenset(v) for k, v in routes.items()}, reason))


heads((1,), 128, 16, 8, 8, 1, "one head, one hidden chunk, C 16 (32-byte swizzle, bk 16), 8x8 map (one tile, half empty)")
heads((16, 17), 256, 32, 8, 9, 3, "two heads (npad 16 / 32), C 32, 8x9 map: partial tile column")
heads((1, 2, 34, 17, 2, 34), 256, 64, 24, 40, 1, "the DLA-34 head set at 24x40")
heads((32, 33, 48, 1, 16, 17, 2, 5), 384, 48, 9, 8, 1, "eight heads, three hidden chunks, C 48 (three bk-16 slabs), 9x8")
heads((1, 16, 17, 32, 33, 48, 2, 3, 5), 128, 64, 17, 23, 3, "nine heads: eight fused, the ninth left as a conv pair")
heads((48, 33), 384, 16, 17, 23, 1, "widest heads (npad 48) with three chunks, C 16")
heads((17,), 256, 48, 24, 40, 3, "one head, C 48, B 3")
heads((2, 32), 128, 32, 9, 8, 1, "9x8: partial tile row")


def heads_program(pb, x, params, outs):
    """the head convs on PlanBuilder ``pb`` over activation ``x``: params[i] = (w3, b3, w1, b1), outs[i] its NCHW output
    Sym"""
    for (w3, b3, w1, b1), o in zip(params, outs):
        h = pb.conv([x], w3, b3, stride=1, pad=1, relu=True)
        pb.conv([h], w1, b1, out="nchw", dst=o)
