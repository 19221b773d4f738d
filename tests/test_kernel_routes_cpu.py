"""CPU checks of the kernel route table and its edge cases (tests/kernel_routes.py): every route has a case, every case
is a call PlanBuilder accepts, the routes a case declares agree with the ops PlanBuilder emits for it, and the library
holds no network-op kernel the table does not name."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from tests.kernel_routes import (CASES, CVT_IN, CVT_OUT, HEAD_CASES, ROUTES, S2D, UNREACHABLE, heads_program,
                                 kernel_key)
from tests.replay import _is_sym, _is_syms

CPU = torch.device("cpu")
TC_KERNELS = ("conv_tc_kernel<", "conv3x3_tc_kernel<", "conv_sp_kernel<", "stem_tc_kernel<", "stem_tc_h_kernel<",
              "heads_tc_kernel<")


def _precision(p):
    return ("bf16", False) if p == "bf16-simt" else (p, None)


def _emit_cpu(case, precision, tc):
    """make the case's call on a CPU PlanBuilder (no data) -> the builder"""
    from centerpose_b200.plan import PlanBuilder
    rec = case.rec
    img = [d for _, d in rec.args if _is_sym(d) and d[4] == "nchw_in"]
    H, W = (img[0][2], img[0][3]) if img else (1, 1)
    pb = PlanBuilder(case.B, H, W, precision, CPU, tc=tc)

    def act(d):
        _, C, h, w, kind, pc, off = d
        s = pb._sym(pc or C, h, w, "act", "external")
        s.fixed = True
        return pb.channel_slice(s, off, C) if pc else s
    kw = {}
    for name, d in rec.args:
        if _is_syms(d):
            kw[name] = [act(s) for s in d]
        elif _is_sym(d) and d[4] == "nchw_in":
            kw[name] = pb.input(d[1])
        elif _is_sym(d) and d[4] == "nchw_out":
            kw[name] = pb.output(d[1], d[2], d[3], "out")
        elif _is_sym(d):
            kw[name] = act(d)
        elif isinstance(d, tuple) and len(d) == 2 and d[0] == "tensor":
            kw[name] = torch.randn(*d[1])
        else:
            kw[name] = d
    getattr(pb, rec.method)(**kw)
    return pb


def test_kernel_key_reads_both_demanglings():
    assert kernel_key("<unnamed>::conv_tc_kernel<(int)64, (bool)0, (int)2>(<unnamed>::TcArgs)") == "conv_tc_kernel<64,false,2>"
    assert kernel_key("void (anonymous namespace)::conv_tc_kernel<64, false, 2>((anonymous namespace)::TcArgs)") == \
        "conv_tc_kernel<64,false,2>"
    assert kernel_key("void (anonymous namespace)::maxpool_kernel<__nv_bfloat16 const*, __nv_bfloat16*>("
                      "__nv_bfloat16 const*, __nv_bfloat16*, int)") == "maxpool_kernel<bf16*,bf16*>"
    assert kernel_key("<unnamed>::convert_to_split_kernel(const float *, unsigned short *, long long)") == CVT_OUT


def test_every_route_has_a_case():
    """... and an exact one"""
    declared, exact = set(), set()
    for c in CASES:
        for p in c.routes:
            declared |= c.routes[p]
            if c.exact and not c.error:
                exact |= c.routes[p]
    for hc in HEAD_CASES:
        for p in hc.routes:
            declared |= hc.routes[p]
            exact |= hc.routes[p]
    assert declared <= set(ROUTES), sorted(declared - set(ROUTES))
    assert set(ROUTES) <= declared, sorted(set(ROUTES) - declared)
    missing = sorted(r for r in ROUTES if r not in exact)
    assert not missing, f"routes without an exact case: {missing}"
    assert not set(UNREACHABLE) & set(ROUTES)


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[f"{i}-{c.rec.method}" for i, c in enumerate(CASES)])
def test_case_routes_agree_with_the_builder(idx):
    from centerpose_b200 import plan as P
    case = CASES[idx]
    assert case.reason
    for pkey, want in case.routes.items():
        for precision in (["bf16x2", "fp16x2"] if pkey == "x2" else [pkey]):
            prec, tc = _precision(precision)
            pb = _emit_cpu(case, prec, tc)
            ops = pb.ops
            tc_ops = [o for o in ops if o.flags & P.FLAG_TC]
            n_tc_routes = sum(1 for k in want if k.startswith(TC_KERNELS))
            assert bool(tc_ops) == (n_tc_routes > 0), (case.label(), precision, [(o.type, o.flags) for o in ops])
            conv = {CVT_IN if o.flags & P.FLAG_TO_F32 else CVT_OUT for o in ops if o.type == P.OP_CONVERT}
            assert conv == want & {CVT_IN, CVT_OUT}, (case.label(), precision, conv)
            assert any(o.type == P.OP_S2D for o in ops) == (S2D in want), (case.label(), precision)
            dcn = [o for o in ops if o.type == P.OP_DCN]
            if dcn:
                assert bool(dcn[0].flags & P.FLAG_TC) == any(",true," in k and k.startswith("conv_tc") for k in want)


@pytest.mark.parametrize("idx", range(len(HEAD_CASES)))
def test_head_cases_fuse(idx):
    from centerpose_b200 import plan as P
    hc = HEAD_CASES[idx]
    for precision in hc.precisions():
        pb = P.PlanBuilder(hc.B, hc.H, hc.W, precision, CPU)
        x = pb._sym(hc.C, hc.H, hc.W, "act", "external")
        x.fixed = True
        x.buf = torch.zeros(1)
        params = [(torch.randn(hc.hid, hc.C, 3, 3), torch.randn(hc.hid), torch.randn(co, hc.hid, 1, 1), torch.randn(co))
                  for co in hc.couts]
        outs = [pb.output(co, hc.H, hc.W, f"head{k}") for k, co in enumerate(hc.couts)]
        heads_program(pb, x, params, outs)
        plan = pb.build()
        fused = [i for i, o in enumerate(plan.pb.ops) if o.type == P.OP_HEADS]
        assert len(fused) == 1
        assert [(e.hidden, e.cout) for e in plan._head_tables[fused[0]]] == [(hc.hid, c) for c in hc.couts[:8]]
        rest = [o for o in plan.pb.ops if o.type != P.OP_HEADS]
        assert len(rest) == 2 * (len(hc.couts) - hc.fused) and all(o.flags & P.FLAG_TC for o in rest)


def _library_kernels():
    from centerpose_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    if not os.path.exists(_lib.LIBPATH):
        pytest.skip("the CUDA library has not been built")
    if not (os.path.exists(tool) and os.path.exists(filt)):
        pytest.skip("cuobjdump / cu++filt not found")
    elf = subprocess.run([tool, "-elf", _lib.LIBPATH], capture_output=True, text=True, check=True).stdout
    # kernels of the anonymous namespaces of csrc/net*.cu: the mangled namespace name carries the source file's name
    mangled = sorted(set(re.findall(r"\.text\.(_Z\S*_net[a-z0-9_]*_cu_\S+)", elf)))
    assert mangled, "no network-op kernels found in the library"
    names = subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout.split("\n")
    return {kernel_key(n) for n in names if n.strip()}


def test_every_library_kernel_has_a_route():
    """A new network-op kernel (or instantiation) fails here until a case runs it."""
    found = _library_kernels()
    unknown = sorted(found - set(ROUTES) - set(UNREACHABLE))
    assert not unknown, f"kernels without a ROUTES entry: {unknown}"
    stale = sorted((set(ROUTES) | set(UNREACHABLE)) - found)
    assert not stale, f"ROUTES entries the library does not hold: {stale}"
