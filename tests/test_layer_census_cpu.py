"""CPU tests (-m "not gpu") of the layer census (tests/layer_census.py): the recording builder sees every op the seven
lowerings and the head emit, every recorded method has a float64 replay reference, the census holds the kernel paths
the op-level replay (tests/test_layer_replay_gpu.py) exists to cover, and the replay's integer-exact legs can tell a
right kernel from a wrong one."""
import inspect
import zlib

import pytest
import torch

from tests.layer_census import ARCHS, NOT_LAYERS, REFERENCES, Record, census, lower_recorded, signatures
from tests.replay import _as_stored, _data, _reference, int_exact

OP_CONV, OP_STEM, OP_DWDECONV_ADD, OP_DCN, OP_UPSAMPLE_ADD, OP_DWCONV, OP_CONVERT, OP_S2D = 1, 2, 4, 5, 7, 8, 11, 12
FLAG_RELU, FLAG_TC, FLAG_HSWISH, FLAG_HSIGMOID, FLAG_RELU6, FLAG_CLIP01 = 1, 8, 16, 32, 128, 256
PRECISIONS = ["fp32", "bf16", "bf16x2", "fp16x2"]


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

    mb = c512["mobilenetv2"] + c128["mobilenetv2"]
    assert any(r.method == "conv" and r.arg("w")[1][2:] == (1, 1) and any(o[1] & FLAG_TC and o[1] & FLAG_RELU6
               for o in r.ops) for r in mb), "mobilenetv2: ReLU6 epilogue on tensor-core 1x1 convs"
    assert any(r.method == "dwconv" and r.ops[-1][0] == OP_DWCONV and r.ops[-1][1] & FLAG_RELU6 for r in mb), \
        "mobilenetv2: ReLU6 on depthwise convs"
    assert any(r.method == "stem" and any(o[1] & FLAG_RELU6 for o in r.ops) for r in mb), "mobilenetv2: ReLU6 stem"
    assert any(r.method == "up_add" and r.arg("b") is not None and r.arg("skip") is not None and r.arg("w")[1] == (32, 1, 2, 2)
               and (r.arg("act"), r.arg("stride"), r.arg("pad")) == ("relu", 2, 0)
               and [o[:2] for o in r.ops] == [(OP_DWDECONV_ADD, FLAG_RELU)] for r in mb), \
        "mobilenetv2: bias form of up_add (k 2, stride 2, pad 0, ReLU, skip) at C 32"
    for co in (80, 160):
        assert any(r.method == "conv" and r.arg("w")[1][0] == co and r.arg("w")[1][2:] == (1, 1)
                   and _syms(r.arg("srcs"))[0][2:4] == (4, 5)
                   and [o[0] for o in r.ops] == [OP_CONVERT, OP_CONV, OP_CONVERT] and not r.ops[1][1] & FLAG_TC
                   for r in c128["mobilenetv2"]), f"mobilenetv2: fp32 island around the {co}-channel 1x1 conv on 4x5"
    gh = c512["ghostnet"] + c128["ghostnet"]
    ghost = [r for r in gh if r.method == "conv" and _tc_ops(r) and r.arg("w")[1][2:] == (1, 1)
             and [s[1] for s in _syms(r.arg("srcs"))] == [16, 16]]
    assert any(r.arg("res") is None for r in ghost) and any(r.arg("res") is not None for r in ghost), \
        "ghostnet: tensor-core 1x1 convs over two 16-channel sources, with and without a residual"
    assert any(r.method == "dwconv" and r.arg("stride") == 2 and r.arg("act") is None for r in gh), \
        "ghostnet: depthwise stride 2 without an activation"
    assert any(r.method == "upsample_add" and r.arg("f") == 1 and r.ops[0][0] == OP_UPSAMPLE_ADD for r in gh), \
        "ghostnet: upsample_add with f = 1"
    se = [r for r in gh if r.method == "conv" and r.arg("act") == "clip01" and _syms(r.arg("srcs"))[0][2:4] == (1, 1)
          and any(o[1] & FLAG_CLIP01 for o in r.ops)]
    assert se, "ghostnet: clip01 SE convs on 1x1 maps"
    assert any(r.method == "scale_add" and r.arg("gate")[2:4] == (1, 1) for r in gh), "ghostnet: scale_add, 1x1 gate"
    assert any(r.method == "resize_bilinear" and r.arg("x")[2:4] == (16, 20) and (r.arg("Ho"), r.arg("Wo")) == (128, 128)
               for r in c128["ghostnet"]), "ghostnet: align-corners resize 16x20 -> 128x128"


def _linear(rec):
    """``rec`` without its epilogue activation"""
    return Record(rec.method, tuple((k, None if k == "act" else False if k == "relu" else v) for k, v in rec.args), ())


@pytest.mark.parametrize("arch", ARCHS)
def test_integer_legs_are_exact_and_reach_the_clamps(arch):
    """The precondition of the replay's "int" legs, over every replayed call in every precision: the float64 reference
    on "int" data is held exactly by the format the result is stored in (so an element-for-element comparison judges
    the kernel, not the rounding), and the linear result of every ReLU6 / clip01 layer reaches both clamp bounds (ReLU6
    with values in between), so a clamp at the wrong place cannot pass.  The DCNs' dyadic data has its own test
    (tests/test_dcn_cases_cpu.py): their float64 reference keeps sigmoid(-200) ~ 1e-87 where the kernels hold 0."""
    refs, n = {}, 0
    for precision in PRECISIONS:
        for rec in signatures(arch, precision):
            if not int_exact(rec) or rec.method == "dcn":
                continue
            if rec.call not in refs:
                data = _data(rec, "int")
                act = dict(rec.args).get("act")
                lin = _reference(_linear(rec), data) if act in ("relu6", "clip01") else None
                refs[rec.call] = (_reference(rec, data), act, lin)
            ref, act, lin = refs[rec.call]
            n += 1
            assert torch.equal(ref, _as_stored(rec, precision, ref)), f"{arch} {precision}: {rec.label()}"
            if lin is not None:
                top = 6 if act == "relu6" else 1
                assert (lin <= 0).any() and (lin >= top).any(), f"{arch} {precision} {act}: {rec.label()}"
                assert act == "clip01" or ((lin > 0) & (lin < top)).any(), f"{arch} {precision} {act}: {rec.label()}"
    assert n


def test_census_records_are_stable():
    """Seeds come from the record's call, so one call replays the same data in every precision and process."""
    a = census("hrnet", "fp16x2", 1, 128, 160)
    b = census("hrnet", "bf16", 1, 128, 160)
    common = {r.call for r in a} & {r.call for r in b}
    assert common
    seeds_a = {r.call: r.seed for r in a}
    assert all(seeds_a[r.call] == r.seed for r in b if r.call in common)
    assert a[0].seed == zlib.crc32(repr(a[0].call).encode())
