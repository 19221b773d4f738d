"""CPU tests (-m "not gpu") of the layer census (tests/layer_census.py): the recording builder sees every op the five
lowerings and the head emit, every recorded method has a float64 replay reference, and the census holds the kernel
paths the op-level replay (tests/test_layer_replay_gpu.py) exists to cover."""
import inspect
import zlib

import pytest

from tests.layer_census import ARCHS, NOT_LAYERS, REFERENCES, census, lower_recorded

OP_CONV, OP_STEM, OP_DCN, OP_CONVERT, OP_S2D = 1, 2, 5, 11, 12
FLAG_TC, FLAG_HSWISH, FLAG_HSIGMOID = 8, 16, 32


def _syms(v):
    return list(v) if isinstance(v, tuple) and v and isinstance(v[0], tuple) else [v]


def test_every_public_builder_method_has_a_replay_reference():
    """A new PlanBuilder layer method fails here until the replay knows how to evaluate it."""
    from centerpose_b200.plan import PlanBuilder
    public = {n for n, v in vars(PlanBuilder).items() if not n.startswith("_") and callable(v)}
    assert NOT_LAYERS <= public, NOT_LAYERS - public
    assert public - NOT_LAYERS == set(REFERENCES), (public - NOT_LAYERS) ^ set(REFERENCES)
    for name in REFERENCES:
        assert inspect.signature(getattr(PlanBuilder, name))


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("precision,H,W", [("fp32", 128, 160), ("bf16", 128, 160), ("bf16x2", 128, 160),
                                           ("fp16x2", 128, 160), ("fp16x2", 512, 512)])
def test_census_covers_the_whole_program(arch, precision, H, W):
    """Every op of the builder's program (before pruning) was emitted inside exactly one outermost recorded call, and
    every recorded method has a replay reference."""
    pb = lower_recorded(arch, precision, 1, H, W)
    assert len(pb.program) == len(pb.ops) > 0
    owner = [None] * len(pb.program)
    for i, (a, b) in enumerate(pb.spans):
        for j in range(a, b):
            assert owner[j] is None, (j, pb.records[owner[j]].label(), pb.records[i].label())
            owner[j] = i
    orphans = [j for j, o in enumerate(owner) if o is None]
    assert not orphans, f"{arch} {precision}: ops {orphans} were emitted outside any recorded PlanBuilder call"
    assert {r.method for r in pb.records} <= set(REFERENCES), {r.method for r in pb.records} - set(REFERENCES)
    assert all(r.ops for r in pb.records), [r.label() for r in pb.records if not r.ops]
    recs = census(arch, precision, 1, H, W)
    assert len(set(recs)) == len(recs) and set(recs) == set(pb.records)
    assert len({r.seed for r in recs}) == len({r.call for r in recs})


def _tc_ops(r, type_=OP_CONV):
    return [o for o in r.ops if o[0] == type_ and o[1] & FLAG_TC]


def _bk(srcs):
    bk = 64
    for s in srcs:
        if s[1] % 64:
            bk = min(bk, 32 if s[1] % 32 == 0 else 16)
    return bk


def _sp_fed(r):
    """a conv the SIMT-fed small-channel kernel runs (csrc/net_tc_sp.cu sp_eligible)"""
    if r.method != "conv" or not _tc_ops(r) or r.arg("out") != "act":
        return False
    srcs = _syms(r.arg("srcs"))
    co, ci, kh, kw = r.arg("w")[1]
    return (len(srcs) == 1 and not srcs[0][5] and srcs[0][1] in (16, 32) and co in (16, 32, 64) and (kh, kw) == (3, 3)
            and r.arg("pad") == 1 and r.arg("stride") in (1, 2))


def test_fp16x2_census_holds_the_kernel_paths_the_replay_covers():
    """The shapes the hand-picked op lists miss, present in the fp16x2 lowerings (presence, not exact counts)."""
    c512 = {a: census(a, "fp16x2", 1, 512, 512) for a in ARCHS}
    c128 = {a: census(a, "fp16x2", 1, 128, 160) for a in ARCHS}
    hd = [r for r in c512["hardnet"] if r.method == "conv" and _tc_ops(r)]
    multi3 = [r for r in hd if len(_syms(r.arg("srcs"))) > 1 and r.arg("w")[1][2] == 3]
    assert multi3, "hardnet: multi-input 3x3 convs on the tensor cores"
    assert any(_bk(_syms(r.arg("srcs"))) == 16 and len({s[1] % 64 for s in _syms(r.arg("srcs"))}) > 1 for r in multi3), \
        "hardnet: multi-input 3x3 convs whose mixed slab widths force BK = 16"
    assert any(r.arg("w")[1][0] % 64 for r in hd if r.arg("out") == "act"), "hardnet: 16-bit outputs with partial N tiles"
    for arch in ("res_50", "hrnet"):
        convs = [r for r in c512[arch] if r.method == "conv" and _tc_ops(r)]
        assert any(r.arg("w")[1][0] == 384 and r.arg("w")[1][2] == 3 for r in convs), f"{arch}: fused head 3x3 conv"
        sliced = [r for r in convs if r.arg("out") == "nchw" and _syms(r.arg("srcs"))[0][5] == 384]
        assert sliced, f"{arch}: channel-slice head 1x1 convs"
    assert any(r.method == "deconv_k4s2" and len(_tc_ops(r)) == 4 for r in c512["res_50"]), "res_50: tensor-core parity convs"
    assert any(r.method == "conv" and any(o[1] & FLAG_TC and o[1] & (FLAG_HSWISH | FLAG_HSIGMOID) for o in r.ops)
               for r in c512["mobilenetv3"]), "mobilenetv3: h-swish / h-sigmoid epilogue on split planes"
    for arch in ("dla_34", "mobilenetv3"):
        assert any(r.method == "dcn" and _tc_ops(r, OP_DCN) for r in c512[arch]), f"{arch}: DCN on the tensor cores"
    for arch in ("res_50", "hrnet", "mobilenetv3", "hardnet"):
        assert any(r.method == "stem" and r.ops[0][0] == OP_S2D for r in c512[arch]), f"{arch}: space-to-depth stem"
    assert any(r.method == "stem" and _tc_ops(r, OP_STEM) for r in c512["dla_34"]), "dla_34: tensor-core stem"
    for arch in ("dla_34", "hrnet", "hardnet"):
        assert any(_sp_fed(r) for r in c512[arch]), f"{arch}: SIMT-fed small-channel conv"
    for arch in ("dla_34", "res_50", "hrnet", "mobilenetv3"):
        assert any(any(o[0] == OP_CONVERT for o in r.ops) for r in c128[arch]), f"{arch}: fp32 islands at 128x160"


def test_census_records_are_stable():
    """Seeds come from the record's call, so one call replays the same data in every precision and process."""
    a = census("hrnet", "fp16x2", 1, 128, 160)
    b = census("hrnet", "bf16", 1, 128, 160)
    common = {r.call for r in a} & {r.call for r in b}
    assert common
    seeds_a = {r.call: r.seed for r in a}
    assert all(seeds_a[r.call] == r.seed for r in b if r.call in common)
    assert a[0].seed == zlib.crc32(repr(a[0].call).encode())
