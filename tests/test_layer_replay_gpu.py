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

Every DCN is replayed twice more, with CPB200_RZ_COMP=0 at plan build (tests/replay.py): on dyadic data, where it must
equal the float64 reference element by element as the output format stores it, and on "coord" data (exact sampling
positions, real-valued samples), held to the conv bounds below rather than the DCN's.

Tolerances (those of tests/test_net_gpu.py, tests/test_split_gpu.py and tests/test_hardnet_gpu.py):
  fp32   : |err| <= 2e-4 max|ref|;  DCN 5e-4 (test_dcn_op_matches_oracle: the sampling positions come from the fp32
           offset conv, whose summation order differs from the reference's)
  bf16   : |err| <= 1e-2 max|ref|;  DCN relative L2 <= 2e-2
  bf16x2 : |err| <= 3e-4 max|ref|
  fp16x2 : |err| <= 1e-5 max|ref|
  split DCN: relative L2 <= 4 tol and |err| <= 40 tol max|ref|  (a sample within rounding of a pixel boundary flips corners)
  max-pool: exact on the values the input planes hold.  upsample_add always adds a skip here, whose sum is rounded
           (fp32, or re-split into planes), so it is held to the precision's bound.

Guards and data: tests/replay.py.
"""
import time

import pytest
import torch

from tests.layer_census import ARCHS, census
from tests.replay import RELU_INPUTS, _data, _judge, _reference, _replay, _stored

pytestmark = pytest.mark.gpu
B = 2
# fp32 / bf16x2 / fp16x2 replay identical data: keep them together so that they share the float64 references
PRECS = ["fp32", "bf16x2", "fp16x2", "bf16"]


def signatures(arch, precision):
    base = census(arch, precision, 1, 128, 160)
    seen = {r.shapeless for r in base}
    extra = [r for r in census(arch, precision, 1, 512, 512) if r.shapeless not in seen]
    return list(base) + list(dict.fromkeys(extra))


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
def test_layer_replay(arch, precision, monkeypatch):
    t0 = time.time()
    recs = signatures(arch, precision)
    split = precision in ("bf16x2", "fp16x2")
    failures, worst, n = [], (-1.0, ""), 0
    for rec in recs:
        variants = ["bf16"] if precision == "bf16" else ["f32"]
        if split and rec.method in RELU_INPUTS:
            variants.append("relu")
        exact_pos = {"int", "coord", "coord-bf16"}
        if rec.method == "dcn":
            variants += ["int", "coord-bf16" if precision == "bf16" else "coord"]
        for variant in variants:
            n += 1
            label = f"{rec.label()} [{variant} inputs]"
            data = _data(rec, variant)
            try:
                with monkeypatch.context() as mp:
                    if variant in exact_pos:
                        mp.setenv("CPB200_RZ_COMP", "0")
                    got, problems = _replay(rec, precision, data)
            except Exception as e:                          # an op the library rejects is a finding too
                failures.append(f"{label}: {type(e).__name__}: {e}")
                continue
            if rec.method == "maxpool":
                from centerpose_b200.plan import PlanBuilder
                pb = PlanBuilder(B, 1, 1, precision, torch.device("cpu"))
                ref = _reference(rec, data, {"x": _stored(pb, data["x"])})
            elif variant in ("bf16", "coord-bf16"):
                ref = _reference(rec, data)
            else:
                ref = _cached_reference(arch, rec, variant, data)
            ratio, ok, how = _judge(rec, precision, got, ref, exact=variant == "int",
                                    positions_exact=variant in ("coord", "coord-bf16"))
            if ratio > worst[0]:
                worst = (ratio, label)
            if problems or not ok:
                failures.append(f"{label}: err/max {ratio:.3e} ({how}){'; ' + '; '.join(problems) if problems else ''}")
    print(f"\n{arch} {precision}: {len(recs)} signatures, {n} replays, worst err/max {worst[0]:.3e} at {worst[1]}"
          f" ({time.time() - t0:.1f} s)")
    assert not failures, f"{arch} {precision}: {len(failures)} of {n} replays failed:\n" + "\n".join(failures)
