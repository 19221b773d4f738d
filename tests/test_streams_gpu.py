"""Every C entry point that takes a stream puts all its work on it (tests/stream_cases.py lists them), and a network
plan orders its runs across streams.

The harness is a held stream.  On a fresh side stream ``s`` the inputs are allocated and given decoy values, a spin
kernel (``torch.cuda._sleep``) is enqueued, and then, still on ``s``, the real inputs are copied in, the entry point is
called through its wrapper and its outputs are cloned.  When the host call returns, the event recorded after the spin
must still be pending: the whole call was enqueued while ``s`` was held.

Decoys are 0xFF bytes (NaN in every float format) for data payloads only: maps, pixels, weights.  Inputs that a
kernel turns into addresses (launch tables, packed files with their tables, gather indices, detection rows that are
sorted) get valid values that give different results, or their real values before the hold: a kernel that escapes its
stream must read in-range addresses and fail an assertion, not fault the device.

* Late escape: the first held leg holds the default stream and leaves ``s`` free.  Work that lands on the default
  stream runs after the clone on ``s``, so the clone misses it, or it overwrites the outputs after the clone.  It runs
  on the real inputs and, since the clones come from another stream's pool, on tables the wrapper has not yet freed
  for reuse.  A launch on the default or legacy stream fails here, before any leg lets it run early.
* Early escape: the second leg holds ``s``.  Work that lands on another stream runs during the spin, on the decoys,
  and its writes to the outputs are overwritten by their poison, which is enqueued on ``s`` after the spin.

Both legs compare the clones, and the outputs after a synchronize, with the same call on the default stream, bit for
bit (the rest of the suite holds that result to its float64 or reference bound).  The outputs the test allocates are
zero-filled on the default stream and 0xFF-filled in the held legs, so each must also be overwritten in full.  The DCN's
grad_input is scattered with fp32 atomics and is compared under tests/test_dcn_train_gpu.py's bound.

``val_targets`` and ``train_batch`` take no device inputs and their wrappers allocate their outputs, so nothing of
theirs is poisoned: only the default-held leg can see them escape.
"""
import ctypes
import math
import os
import random
import time

import numpy as np
import pytest
import torch

from centerpose_b200 import _lib
from tests.stream_cases import HELD, PLAN_FAMILIES, SYNCED

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
HOLD_S = 0.2                       # seconds of spin in a held leg
MEAN = (0.408, 0.447, 0.470)
STD = (0.289, 0.274, 0.278)
_CYCLES = {}                       # device index -> spin cycles per millisecond
_MODELS = {}


def _cycles(dev, seconds):
    """``torch.cuda._sleep`` cycles that spin about ``seconds`` on ``dev`` (timed once per device with events)."""
    if dev.index not in _CYCLES:
        with torch.cuda.device(dev):
            torch.cuda._sleep(1000)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            torch.cuda._sleep(20_000_000)
            b.record()
            b.synchronize()
            _CYCLES[dev.index] = 20_000_000 / a.elapsed_time(b)
    return int(_CYCLES[dev.index] * seconds * 1000)


class Alloc:
    """Allocates a call's outputs on the current stream: zero-filled on the default-stream leg, 0xFF-filled in the
    held legs.  ``poison=False`` zero-fills in every leg (an output the entry point writes only in part by design)."""

    def __init__(self, dev, value):
        self.dev, self.value = dev, value

    def __call__(self, shape, dtype, poison=True):
        t = torch.empty(shape, dtype=dtype, device=self.dev)
        t.view(-1).view(torch.uint8).fill_(self.value if poison else 0)
        return t


KEEP = "keep"                      # a decoy: the input holds its real values before the hold too


class Case:
    """``inputs``: device tensors holding the real input values.  ``call(ins, alloc)`` enqueues the entry point on
    the current stream with ``ins`` (copies of ``inputs``, or ``inputs`` themselves when ``inplace``: a plan bakes its
    input addresses in) and returns its outputs.  ``decoys[i]``: what input i holds before the hold; None is 0xFF
    bytes (data payloads only), KEEP its real values, a tensor other valid values.  ``loose``: indices of outputs
    compared under the atomics bound."""

    def __init__(self, inputs, call, inplace=False, loose=(), decoys=None):
        self.inputs, self.call, self.inplace, self.loose = list(inputs), call, inplace, set(loose)
        self.saved = [t.clone() for t in self.inputs] if inplace else self.inputs
        self.decoys = list(decoys) if decoys is not None else [None] * len(self.inputs)
        assert len(self.decoys) == len(self.inputs)


def _fill(t, value):
    t.view(-1).view(torch.uint8).fill_(value)


def _decoy(b, d, real):
    if d is None:
        _fill(b, 0xFF)
    else:
        b.copy_(real if d is KEEP else d)


def run_leg(case, dev, hold=None, guard=True):
    """One call of ``case`` on ``dev``: on the default stream (``hold`` None), or on a side stream with that stream
    (``"side"``) or the default stream (``"default"``) held.  Returns (clones taken on the call's stream, outputs).
    ``guard=False`` makes the default-stream call with the current device left as it is."""
    with torch.cuda.device(dev if guard else None):
        if hold is None:
            ins = case.inputs if case.inplace else [t.clone() for t in case.inputs]
            outs = case.call(ins, Alloc(dev, 0))
            clones = [o.clone() for o in outs]
            torch.cuda.synchronize(dev)
            return clones, outs
        s = torch.cuda.Stream(dev)
        held = s if hold == "side" else torch.cuda.default_stream(dev)
        e_held = torch.cuda.Event()
        with torch.cuda.stream(s):
            ins = case.inputs if case.inplace else [torch.empty_like(t) for t in case.inputs]
            for b, d, t in zip(ins, case.decoys, case.saved):
                _decoy(b, d, t)
        if hold == "default":
            torch.cuda.synchronize(dev)           # the decoys are in place before the call may touch the inputs
        with torch.cuda.stream(held):
            torch.cuda._sleep(_cycles(dev, HOLD_S))
            e_held.record()
        with torch.cuda.stream(s):
            for b, d, t in zip(ins, case.decoys, case.saved):
                if d is not KEEP:
                    b.copy_(t)
            outs = case.call(ins, Alloc(dev, 0xFF))
        # the clones' memory comes from another stream's pool: taking a clone on s must not reuse a block the wrapper
        # freed on s (a launch table) while work that escaped to the held default stream has yet to read it
        with torch.cuda.stream(torch.cuda.Stream(dev)):
            clones = [torch.empty_like(o, memory_format=torch.contiguous_format) for o in outs]
        with torch.cuda.stream(s):
            for c, o in zip(clones, outs):
                c.copy_(o)
                c.record_stream(s)
        pending = not e_held.query()
        torch.cuda.synchronize(dev)
    assert pending, ("the %s stream's %.2f s hold ended before the call returned: lengthen HOLD_S (the call's host "
                     "time exceeds it, or it synchronized)" % (hold, HOLD_S))
    return clones, outs


def _bytes(t):
    return t.detach().contiguous().view(-1).view(torch.uint8)


def same(got, want, label, loose=()):
    assert len(got) == len(want), label
    bad = []
    for k, (g, w) in enumerate(zip(got, want)):
        if g.shape != w.shape or g.dtype != w.dtype:
            bad.append("output %d: %s %s, expected %s %s" % (k, tuple(g.shape), g.dtype, tuple(w.shape), w.dtype))
        elif k in loose:
            scale = w.abs().max().item()
            err = (g.double() - w.double()).nan_to_num(float("inf")).abs().max().item()
            if not err <= 1e-6 * scale:
                bad.append("output %d: max |diff| %.3g > 1e-6 * %.3g" % (k, err, scale))
        elif not torch.equal(_bytes(g), _bytes(w)):
            n = int((_bytes(g) != _bytes(w)).sum())
            nan = int(g.isnan().sum()) if g.is_floating_point() else 0
            bad.append("output %d: %d of %d bytes differ (%d NaN)" % (k, n, _bytes(g).numel(), nan))
    assert not bad, label + ":\n" + "\n".join(bad)


def check_held(case, dev):
    want, _ = run_leg(case, dev)
    for hold in ("default", "side"):
        clones, outs = run_leg(case, dev, hold)
        same(clones, want, "%s stream held: the clone taken on the call's stream" % hold, case.loose)
        same(outs, want, "%s stream held: the outputs after synchronize" % hold, case.loose)


# --------------------------------------------------------------------------------------------------- network plans
def _family(fam):
    """The first case of tests/kernel_routes.py of kernel family ``fam`` with bf16 and split routes."""
    from tests.kernel_routes import CASES, CVT_IN

    def k(c):
        w = dict(c.rec.args).get("w")
        return tuple(w[1][2:]) if w else None

    def tc(c, dcn):
        return any(x.startswith("conv_tc_kernel<") and (",true," in x) == dcn for r in c.routes.values() for x in r)

    def has(c, prefix):
        return any(x.startswith(prefix) for r in c.routes.values() for x in r)

    pred = {"tap": lambda c: c.rec.method == "conv" and k(c) == (3, 3) and tc(c, False),
            "pointwise": lambda c: c.rec.method == "conv" and k(c) == (1, 1) and dict(c.rec.args)["stride"] == 1
            and tc(c, False),
            "halo": lambda c: c.rec.method == "conv" and has(c, "conv3x3_tc_kernel<"),
            "small_channel": lambda c: c.rec.method == "conv" and has(c, "conv_sp_kernel<"),
            "stem": lambda c: c.rec.method == "stem" and has(c, "stem_tc"),
            "dcn": lambda c: c.rec.method == "dcn" and tc(c, True),
            "eltwise": lambda c: c.rec.method == "maxpool",
            "convert": lambda c: CVT_IN in c.routes.get("x2", ())}[fam]
    return next(c for c in CASES if not c.error and "bf16" in c.routes and "x2" in c.routes and pred(c))


def _plan_case(fam, precision, dev):
    from centerpose_b200.plan import PlanBuilder
    if fam == "heads":
        return _heads_case(precision, dev)
    from tests.replay import _data, _emit, _is_sym
    c = _family(fam)
    img = [d for _, d in c.rec.args if _is_sym(d) and d[4] == "nchw_in"]
    H, W = (img[0][2], img[0][3]) if img else (1, 1)
    pb = PlanBuilder(c.B, H, W, precision, dev)
    y, img_buf, ch_off = _emit(pb, c.rec, _data(c.rec, "bf16" if precision == "bf16" else "f32", c.B))
    nchw = y.kind == "nchw_out"
    if not nchw:
        pb.keep_result(y)
    plan = pb.build()
    ext = {}
    for po in plan.pb.ops:
        for s in po.operands():
            r = plan._root(s)
            if r.fixed and r.kind == "act":
                ext[id(r.buf)] = r.buf
    inputs = ([img_buf] if img_buf is not None else []) + list(ext.values())
    root = plan._root(y)

    def call(ins, alloc):
        if nchw:
            out = alloc((c.B, y.C, y.H, y.W), torch.float32)
            plan.bind(img_buf, {"out": out})
            plan.run()
            return [out[:, ch_off:ch_off + y.C - 4]]
        if img_buf is not None:
            plan.bind(img_buf, {})
        region = root.buf.view(-1)[:c.B * root.H * root.W * root.C * pb._storage(root.kind)[0]]
        region.fill_(alloc.value)
        plan.run()
        return [region]
    # a DCN samples at offsets computed from its input: a valid decoy, not NaN
    decoys = [t * 0.5 for t in inputs] if fam == "dcn" else None
    return Case(inputs, call, inplace=True, decoys=decoys)


def _heads_case(precision, dev):
    from centerpose_b200.plan import PlanBuilder
    from tests.kernel_routes import HEAD_CASES, heads_program
    from tests.replay import _place_act
    from tests.test_kernel_envelope_gpu import _head_params
    hc = HEAD_CASES[1]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(hc.B, hc.C, hc.H, hc.W, generator=g)
    params = _head_params(hc, "f32", g)
    pb = PlanBuilder(hc.B, hc.H, hc.W, precision, dev)
    xs = _place_act(pb, x, ("sym", hc.C, hc.H, hc.W, "act", 0, 0))
    heads_program(pb, xs, params, [pb.output(co, hc.H, hc.W, "head%d" % k) for k, co in enumerate(hc.couts)])
    plan = pb.build()

    def call(ins, alloc):
        outs = {"head%d" % k: alloc((hc.B, co, hc.H, hc.W), torch.float32) for k, co in enumerate(hc.couts)}
        plan.bind(None, outs)
        plan.run()
        return list(outs.values())
    return Case([xs.buf], call, inplace=True)


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The DLA-34 models (and their cached plans) the module's tests share are dropped when the module ends."""
    yield
    _MODELS.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _dla34(dev):
    if dev.index not in _MODELS:
        from tests.util import model
        m, _ = model("dla_34", "fp16x2")
        _MODELS[dev.index] = m.to(dev)
    return _MODELS[dev.index]


def _model_case(dev):
    from tests.util import golden_input
    m = _dla34(dev)
    x = golden_input("dla34_96x160").to(dev)
    # the DCNs sample at offsets the network computes from the input: a valid decoy, not NaN
    return Case([x], lambda ins, alloc: list(m(ins[0])), decoys=[x * 0.5])


# --------------------------------------------------------------------------------------------- decode and post
def _maps(dev, B=2, J=17, H=24, W=40, seed=3):
    g = torch.Generator().manual_seed(seed)
    t = [torch.rand(B, 1, H, W, generator=g), torch.rand(B, 2, H, W, generator=g) * 20,
         torch.randn(B, 2 * J, H, W, generator=g) * 5, torch.rand(B, 2, H, W, generator=g),
         torch.rand(B, J, H, W, generator=g), torch.rand(B, 2, H, W, generator=g)]
    return [x.to(dev) for x in t]


def _decode_case(dev, affine=False):
    from centerpose_b200 import multi_pose_decode
    ins, decoys = _maps(dev), _maps(dev, seed=4)          # top-K selection on NaN maps is not defined: valid decoys
    if affine:
        ins.append(torch.tensor([[4.0, 0.5, 3.0, -0.25, 4.0, 7.0], [2.0, 0.0, -5.0, 0.0, 2.0, 1.0]], device=dev))
        decoys.append(None)

    def call(x, alloc):
        return [multi_pose_decode(x[0], x[1], x[2], reg=x[3], hm_hp=x[4], hp_offset=x[5], K=50,
                                  affine=x[6] if affine else None)]
    return Case(ins, call, decoys=decoys)


def _sigmoid_case(dev):
    from centerpose_b200.decode import sigmoid_
    x = torch.randn(3, 17, 33, 29, generator=torch.Generator().manual_seed(1)).to(dev) * 4
    return Case([x], lambda ins, alloc: [sigmoid_(ins[0])])


def _boxes(B, N, seed):
    rng = np.random.default_rng(seed)
    b = np.zeros((B, N, 56), np.float32)
    xy = rng.uniform(0, 100, (B, N, 2))
    wh = rng.uniform(5, 40, (B, N, 2))
    b[..., 0:2], b[..., 2:4] = xy, xy + wh
    b[..., 4] = rng.uniform(0, 1, (B, N))
    b[..., 5:39] = rng.uniform(0, 140, (B, N, 34))
    b[..., 39:56] = rng.uniform(0, 1, (B, N, 17))
    return torch.from_numpy(b)


def _soft_nms_case(dev):
    def call(ins, alloc):
        keep = alloc((1,), torch.int32)
        _lib.launch("soft_nms_39", dev, ins[0], ins[0].shape[0], 0.5, 0.3, 0.001, 2, keep)
        return [ins[0], keep]
    return Case([_boxes(1, 60, 1)[0].to(dev)], call)


def _soft_nms_batch_case(dev):
    from centerpose_b200.soft_nms import soft_nms_39_cuda_batch
    return Case([_boxes(3, 50, 2).to(dev)], lambda ins, alloc: [ins[0], soft_nms_39_cuda_batch(ins[0], method=1)])


def _flip_case(dev):
    from centerpose_b200.decode import flip_merge
    ins = _maps(dev, B=4, seed=5)
    flip_idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    return Case([ins[0], ins[1], ins[2], ins[4]],
                lambda x, alloc: list(flip_merge(x[0], x[1], x[2], x[3], flip_idx)))


def _image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _host_floats(ctype, vals):
    return (ctype * len(vals))(*vals)


def _trans(h, w, oh, ow):
    from centerpose_b200.image import get_affine_transform
    c = np.array([w / 2.0, h / 2.0], np.float32)
    return np.asarray(get_affine_transform(c, max(h, w) * 1.0, 0, [ow, oh]), np.float64).reshape(6)


def _pre_process_case(dev):
    h, w, oh, ow = 37, 53, 64, 64
    M = _host_floats(ctypes.c_double, _trans(h, w, oh, ow).tolist())

    def call(ins, alloc):
        out = alloc((2, 3, oh, ow), torch.float32)
        _lib.launch("pre_process", dev, ins[0], h, w, M, out, oh, ow, _host_floats(ctypes.c_float, MEAN),
                    _host_floats(ctypes.c_float, STD), 1)
        return [out]
    return Case([torch.from_numpy(_image(h, w, 3)).to(dev)], call)


def _pre_process_batch_case(dev, f32):
    from centerpose_b200.detector import _PRE_IMAGE
    shapes, oh, ow = [(37, 53), (64, 20)], 32, 64
    imgs = [_image(h, w, 4 + k) for k, (h, w) in enumerate(shapes)]
    table = np.zeros(len(shapes), _PRE_IMAGE)
    off = 0
    for e, (h, w) in zip(table, shapes):
        e["offset"], e["h"], e["w"], e["trans_input"] = off, h, w, _trans(h, w, oh, ow)
        off += h * w * 3
    pixels = torch.from_numpy(np.concatenate([i.reshape(-1) for i in imgs])).to(dev)
    tab = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).to(dev)
    B = len(shapes)

    def call(ins, alloc):
        mean, std = _host_floats(ctypes.c_float, MEAN), _host_floats(ctypes.c_float, STD)
        if f32:
            out = alloc((B, 3, oh, ow), torch.float32)
            _lib.launch("pre_process_batch_f32", dev, ins[0], ins[1], B, out, oh, ow, mean, std)
        else:
            out = alloc((2 * B, 3, oh, ow), torch.float32)
            _lib.launch("pre_process_batch", dev, ins[0], ins[1], B, out, oh, ow, mean, std, 1)
        return [out]
    return Case([pixels, tab], call, decoys=[None, KEEP])


def _resize_case(dev):
    from centerpose_b200.detector import resize_table
    shapes, new = [(37, 53), (20, 64)], [(50, 75), (9, 31)]
    table = resize_table(shapes, new)
    pixels = torch.from_numpy(np.concatenate([_image(h, w, 7 + k).reshape(-1) for k, (h, w) in enumerate(shapes)]))
    n = sum(h * w * 3 for h, w in new)

    def call(ins, alloc):
        dst = alloc((n,), torch.uint8)
        _lib.launch("resize_linear_u8_batch", dev, ins[0], ins[1], len(shapes), dst)
        return [dst]
    return Case([pixels.to(dev), torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).to(dev)], call,
                decoys=[None, KEEP])


# ------------------------------------------------------------------------------------------ image files and views
def _files(fmt):
    import cv2
    from tests.test_jpeg_cpu import encode, make_image
    if fmt == "jpeg":
        return [encode(make_image(37, 53, "smooth_noise", 5), 90), encode(make_image(16, 24, "noise", 6), 50, "444")]
    if fmt == "png":
        return [cv2.imencode(".png", make_image(h, w, "smooth_noise", h))[1].tobytes() for h, w in ((37, 53), (9, 70))]
    if fmt == "webp":
        from tests.test_webp_cpu import lossy
        return [lossy(37, 53, 5), lossy(17, 33, 6, 95, "noise")]
    from tests.test_webp_lossless_cpu import lossless
    return [lossless(37, 53, 5), lossless(17, 15, 6, "noise")]


def _decoder_case(fmt, dev):
    from centerpose_b200 import jpeg, png, webp, webp_lossless
    mod = {"jpeg": jpeg, "png": png, "webp": webp, "webp_lossless": webp_lossless}[fmt]
    datas = _files(fmt)
    infos = [mod.parse(d) for d in datas]
    assert all(i.eligible for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = mod.pack(infos, datas, offs[:-1])

    def call(ins, alloc):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        dst, status = alloc((int(offs[-1]),), torch.uint8), alloc((len(datas),), torch.int32)
        _lib.launch(mod.KERNEL, dev, ins[0], ins[0], len(datas), ws, ws_bytes, dst, status)
        return [dst, status]
    return Case([torch.from_numpy(buf).to(dev)], call, decoys=[KEEP])      # the files' bytes and their tables


def _png_encode_case(dev):
    from centerpose_b200 import png
    shapes = [(37, 53), (5, 200)]
    imgs = [torch.from_numpy(_image(h, w, 20 + h)).to(dev) for h, w in shapes]

    def call(ins, alloc):
        table, counts, ws, out_bytes = png.encode_layout([t.data_ptr() for t in ins], shapes, [3 * w for _, w in shapes])
        out = alloc((out_bytes,), torch.uint8, poison=False)       # written up to the files' total only
        sizes = alloc((len(shapes),), torch.int64)
        png.encode_launch(table, counts, ws, out, sizes)
        return [out, sizes]
    return Case(imgs, call)


def _heatmap_case(dev):
    from centerpose_b200 import heatmaps
    g = torch.Generator().manual_seed(8)
    dr, h, w = 4, 12, 10
    ins = [torch.randn(3, h * dr, w * dr, generator=g), torch.rand(1, h, w, generator=g) ** 4,
           torch.rand(17, h, w, generator=g) ** 6]

    def call(x, alloc):
        sizes = heatmaps.check([x[0]], [x[1]], [x[2]], dr)
        table, _, ws = heatmaps.layout([(x[0].data_ptr(), x[1].data_ptr(), x[2].data_ptr())], sizes, dr)
        out = alloc((heatmaps.view_bytes(h * dr, w * dr),), torch.uint8)
        heatmaps.launch(table, ws, "white", np.array(MEAN), np.array(STD), out)
        return [out]
    return Case([t.to(dev) for t in ins], call)


def _render_case(dev):
    from centerpose_b200 import render
    from tests import render_cases as rc
    h, w = 120, 160
    ops = render.build([(h, w)], [rc.rows(h, w, 6, 31)], 0.3, "white")

    def call(ins, alloc):
        render.launch(ops, pixels=ins[0], offsets=[0])
        return [ins[0]]
    return Case([torch.from_numpy(rc.image(h, w, 30).reshape(-1).copy()).to(dev)], call)


# ------------------------------------------------------------------------------------- evaluation and training
def _coco_case(dev, what):
    from centerpose_b200 import coco_eval
    from centerpose_b200.coco_eval import KeypointEval
    from tests.coco_eval_cases import make_case
    gt, res = make_case(3, n_images=8, max_rows=40)
    ev = KeypointEval(gt, device=dev)
    evaluated, _, up, rows, n_rows, n_keep, n_oks = ev._pack(res, None)
    T, R, A = coco_eval.T, coco_eval.R, coco_eval.A

    def call(ins, alloc):
        ws = ev._workspace(len(evaluated), n_rows, n_keep, n_oks)
        if what == "oks":
            out = alloc((max(n_oks, 1),), torch.float64)
            _lib.launch("coco_kp_oks", dev, ins[0], len(evaluated), ins[1], n_rows, ev.gts, ev.n_gts, n_keep, n_oks,
                        ctypes.byref(ev.params), out, ws)
        else:
            out = alloc((2 * T * R * A + T * A,), torch.float64)
            p = out.data_ptr()
            _lib.launch("coco_kp_eval", dev, ins[0], len(evaluated), ins[1], n_rows, ev.gts, ev.n_gts, n_keep, n_oks,
                        ctypes.byref(ev.params), p, p + 8 * 2 * T * R * A, p + 8 * T * R * A, ws)
        return [out]
    return Case([up, rows], call, decoys=[KEEP, rows * 0.5])   # the launch table; rows that are sorted by score


def _target_decoys(ts):
    """Float targets take the 0xFF decoy; gather indices and masks take zeros, an index in range with its mask off."""
    return [None if t.is_floating_point() else torch.zeros_like(t) for t in ts]


def _val_setup(dev):
    from centerpose_b200.coco_eval import KeypointEval
    from centerpose_b200.config import default_cfg
    from tests.val_cases import constructed, shapes_of
    ds = constructed()
    ev = KeypointEval(ds, device=dev)
    sh = shapes_of(ds)
    ids = [im["id"] for im in ds["images"]]
    return default_cfg("dla_34"), ev, ids, [sh[i] for i in ids]


def _val_targets_case(dev):
    from centerpose_b200 import val
    cfg, ev, ids, shapes = _val_setup(dev)
    return Case([], lambda ins, alloc: list(val.targets(ev, ids, shapes, cfg).values()))


def _val_loss_case(dev):
    from centerpose_b200 import val
    from tests.train_loss_cases import logits
    cfg, ev, ids, shapes = _val_setup(dev)
    with torch.cuda.device(dev):
        tg = val.targets(ev, ids, shapes, cfg)
    heads = [torch.from_numpy(h).to(dev) for h in logits(5, len(ids), int(cfg.MODEL.OUTPUT_RES))]
    keys = list(tg)
    return Case(heads + [tg[k] for k in keys],
                lambda ins, alloc: [val.loss(ins[:6], dict(zip(keys, ins[6:])), cfg)],
                decoys=[None] * 6 + _target_decoys([tg[k] for k in keys]))


def _radius_case(dev):
    hw = torch.tensor([(h, w) for h in range(1, 40, 3) for w in range(1, 40, 2)], dtype=torch.int32, device=dev)

    def call(ins, alloc):
        out = alloc((len(hw),), torch.int32)
        _lib.launch("gaussian_radius", dev, ins[0], len(hw), out)
        return [out]
    return Case([hw], call, decoys=[hw + 1])


def _train_batch_case(dev):
    from centerpose_b200 import train_data
    from centerpose_b200.config import default_cfg
    from oracle.make_golden_val import image
    from tests.train_cases import case_cfg, small_case
    cfg = case_cfg(default_cfg("dla_34"), {"FLIP": 1.}, 128)
    ds = small_case()
    pix = [image(4000 + im["id"], im["height"], im["width"]) for im in ds["images"]]
    ids = [im["id"] for im in ds["images"]]
    with torch.cuda.device(dev):
        tr = train_data.TrainData(cfg, ds)

    def call(ins, alloc):
        np.random.seed(5)
        random.seed(15)
        tr.draws.data_rng = np.random.RandomState(123)
        return list(tr.batch(pix, ids).values())
    return Case([], call)


def _train_loss_case(dev):
    from centerpose_b200 import train_loss, val
    from centerpose_b200.config import default_cfg
    from tests import train_loss_cases as tc
    cfg, batch, heads, grad_out = tc.case("shared_pixels", default_cfg("dla_34"))
    keys = list(batch)
    loss = train_loss.MultiPoseLoss(cfg)
    inputs = [torch.from_numpy(np.ascontiguousarray(h)).to(dev) for h in heads] + \
        [torch.from_numpy(np.ascontiguousarray(batch[k])).to(dev) for k in keys]

    def call(ins, alloc):
        hs = [h.requires_grad_(True) for h in ins[:6]]
        lo, stats = loss(hs, dict(zip(keys, ins[6:])))
        lo.backward(torch.full((), grad_out, dtype=torch.float32, device=dev))
        return [lo.detach()] + [stats[k].detach() for k in val.STATS] + [h.grad for h in hs if h.grad is not None]
    return Case(inputs, call, decoys=[None] * 6 + _target_decoys(inputs[6:]))


def _dcn_case(dev, precision):
    from centerpose_b200 import dcn
    from tests.test_dcn_train_gpu import make_inputs
    t = make_inputs(2, 16, 24, 9, 11, seed=4)
    names = ("input", "offset", "mask", "weight", "bias", "grad_out")

    def call(ins, alloc):
        leaves = [x.requires_grad_(True) for x in ins[:5]]
        out = dcn.dcn_v2_conv(*leaves, 1, 1, 1, 1, precision=precision)
        out.backward(ins[5])
        return [out.detach()] + [x.grad for x in leaves]
    ins = [t[n].to(dev) for n in names]
    # sampling positions come from the offsets: zero offsets, not NaN ones, before the hold
    return Case(ins, call, loose=(1,), decoys=[None, torch.zeros_like(ins[1]), None, None, None, None])


BUILD = {
    "model_dla34": _model_case,
    "decode": _decode_case,
    "decode_affine": lambda dev: _decode_case(dev, affine=True),
    "sigmoid": _sigmoid_case,
    "soft_nms": _soft_nms_case,
    "soft_nms_batch": _soft_nms_batch_case,
    "flip_merge": _flip_case,
    "pre_process": _pre_process_case,
    "pre_process_batch": lambda dev: _pre_process_batch_case(dev, False),
    "pre_process_batch_f32": lambda dev: _pre_process_batch_case(dev, True),
    "resize": _resize_case,
    **{f: (lambda dev, f=f: _decoder_case(f, dev)) for f in ("jpeg", "png", "webp", "webp_lossless")},
    "png_encode": _png_encode_case,
    "heatmap_views": _heatmap_case,
    "render_poses": _render_case,
    "coco_kp_oks": lambda dev: _coco_case(dev, "oks"),
    "coco_kp_eval": lambda dev: _coco_case(dev, "eval"),
    "val_targets": _val_targets_case,
    "gaussian_radius": _radius_case,
    "val_loss": _val_loss_case,
    "train_batch": _train_batch_case,
    "train_loss": _train_loss_case,
    "dcn_default": lambda dev: _dcn_case(dev, "default"),
    "dcn_fp32": lambda dev: _dcn_case(dev, "fp32"),
}
PLAN_IDS = [("plan_" + f, p) for f in PLAN_FAMILIES for p in ("bf16", "fp16x2")]


def test_every_case_has_a_builder():
    assert set(BUILD) | {n for n, _ in PLAN_IDS} == set(HELD)


@pytest.mark.parametrize("name,precision", PLAN_IDS, ids=["%s-%s" % c for c in PLAN_IDS])
def test_plan_on_held_stream(name, precision):
    check_held(_plan_case(name[len("plan_"):], precision, DEV), DEV)


@pytest.mark.parametrize("name", sorted(BUILD))
def test_entry_point_on_held_stream(name):
    check_held(BUILD[name](DEV), DEV)


# ------------------------------------------------------------------------------ wrappers that wait for the device
def _same_tree(a, b, what):
    if isinstance(a, dict):
        assert list(a) == list(b), what
        for k in a:
            _same_tree(a[k], b[k], "%s[%r]" % (what, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for k, (x, y) in enumerate(zip(a, b)):
            _same_tree(x, y, "%s[%d]" % (what, k))
    elif isinstance(a, torch.Tensor):
        assert torch.equal(_bytes(a), _bytes(b)), what
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what
    elif isinstance(a, float) and math.isnan(a):
        assert math.isnan(b), what
    else:
        assert a == b, what


def _on_side_stream(fn):
    """``fn()`` on the default stream, then under a side stream: the two results must be equal, bit for bit."""
    want = fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        got = fn()
    torch.cuda.synchronize()
    return got, want


@pytest.mark.parametrize("name", sorted(SYNCED))
def test_synced_wrapper_on_side_stream(name):
    """These wrappers download their results before they return, which uses up any hold, so they take only the
    equality leg: called under a side stream, they return what they return on the default stream."""
    if name == "KeypointEval.evaluate":
        from centerpose_b200.coco_eval import KeypointEval
        from tests.coco_eval_cases import make_case
        gt, res = make_case(4, n_images=8, max_rows=40)
        ev = KeypointEval(gt)

        def fn():
            stats = ev.evaluate(res)
            return [list(stats), {k: ev.eval[k] for k in ("precision", "recall", "scores")}]
    elif name == "run_images":
        from tests.test_jpeg_cpu import make_image
        from tests.test_jpeg_gpu import _detector
        det = _detector("dla_34", "fp16x2", [1.0])
        images = [make_image(96, 128, "smooth_noise", 1), make_image(120, 80, "smooth", 2)]

        def fn():
            return det.run_images(images)
    else:
        from centerpose_b200.coco_eval import KeypointEval
        from centerpose_b200.config import default_cfg
        from centerpose_b200.detector import detector_factory
        from oracle import make_golden_val as g
        from oracle.init_recipe import conditioned_state_dict
        f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "val_dla34.npz"))
        pixels = [g.image(seed, h, w) for seed, h, w in g.VAL_IMAGES]
        cfg = default_cfg("dla_34")
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        ev = KeypointEval(g.dla34_case())
        ids = f["image_ids"].tolist()

        def fn():
            log, preds = det.run_val(pixels, ids, ev, max_batch=2)
            log.pop("time")
            return [log, preds]
    got, want = _on_side_stream(fn)
    _same_tree(got, want, name)


# ------------------------------------------------------------------------------------ one plan, several streams
def _hold(stream, seconds=HOLD_S):
    """A spin of ``seconds`` on ``stream``; returns the event recorded after it."""
    e = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(_cycles(DEV, seconds))
        e.record()
    return e


def _inputs(seed, H=64, W=96, B=1):
    from centerpose_b200.synth import synth_images
    return synth_images(B, H, W, seed).to(DEV)


def test_plan_runs_are_ordered_across_streams():
    """model(x1) on a held stream A, then model(x2) on stream B with no sync between them: both runs use one plan's
    activation buffers, so B's run must wait for A's.  While A's hold is pending, B's end event must not complete, and
    both outputs must equal their default-stream results bit for bit."""
    m = _dla34(DEV)
    x1, x2 = _inputs(1), _inputs(2)
    want1, want2 = [[t.clone() for t in m(x)] for x in (x1, x2)]
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    with torch.cuda.stream(a):
        xa = x1 * 0.5                            # a valid decoy: the DCNs sample at offsets computed from it
    e_a = _hold(a)
    with torch.cuda.stream(a):
        xa.copy_(x1)
        o1 = m(xa)
    with torch.cuda.stream(b):
        o2 = m(x2)
        e_b = torch.cuda.Event()
        e_b.record()
    polls, t0 = 0, time.time()
    while not e_a.query() and time.time() - t0 < 2 * HOLD_S:
        assert not e_b.query(), "the run on stream B finished while the run on stream A was still held"
        polls += 1
        time.sleep(0.002)
    assert polls > 0, "stream A's hold ended before the runs were enqueued: lengthen HOLD_S"
    torch.cuda.synchronize()
    same(o1, want1, "the run on stream A")
    same(o2, want2, "the run on stream B")


def test_evicted_plan_memory_outlives_its_held_run():
    """A plan built on the default stream runs on a held stream A; nine more shapes then evict it from the model's
    cache.  While A's run is pending, allocations on the default stream must not be handed the evicted plan's memory,
    and A's outputs must equal the default-stream result bit for bit."""
    m = _dla34(DEV)
    m.invalidate()
    x0 = _inputs(3)
    want = [t.clone() for t in m(x0)]
    torch.cuda.synchronize()
    (plan,) = m._plans.values()
    spans = [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()) for t in plan.buffers]
    sizes = [t.numel() * t.element_size() for t in plan.buffers]
    del plan
    for k in range(1, 9):                          # eight more shapes: nine plans cached, the next one evicts them
        x = _inputs(3, H=64, W=96 + 32 * k)
        torch.cuda.synchronize()
        t0 = time.time()
        m(x)
        build = time.time() - t0                   # host time of a forward that builds its plan: the tenth's too
    x9 = _inputs(3, H=64, W=96 + 32 * 9)
    torch.cuda.synchronize()
    a = torch.cuda.Stream(DEV)
    with torch.cuda.stream(a):
        xa = x0 * 0.5                            # a valid decoy: the DCNs sample at offsets computed from it
    hold = min(0.5, max(HOLD_S, 3 * build + 0.1))
    print("plan build %.3f s, hold %.3f s" % (build, hold))
    e_a = _hold(a, seconds=hold)
    with torch.cuda.stream(a):
        xa.copy_(x0)
        outs = m(xa)
    m(x9)                                           # the tenth shape: the cache is cleared and the first plan dropped
    assert len(m._plans) == 1
    fresh = [torch.empty(n, dtype=torch.uint8, device=DEV) for n in sizes]
    for t in fresh:
        t.fill_(0xFF)
    pending = not e_a.query()
    overlap = [(t.data_ptr(), lo) for t in fresh for lo, hi in spans
               if t.data_ptr() < hi and lo < t.data_ptr() + t.numel()]
    torch.cuda.synchronize()
    assert pending, "stream A's %.2f s hold ended before the eviction (plan build %.2f s)" % (hold, build)
    assert not overlap, "%d allocations were handed memory of the evicted plan while its run was pending" % len(overlap)
    same(outs, want, "the held run of the evicted plan")
    del fresh, outs


# -------------------------------------------------------------------------------------------------- second device
TWO = torch.cuda.is_available() and torch.cuda.device_count() >= 2


@pytest.mark.skipif(not TWO, reason="one CUDA device: the second-device leg needs two")
@pytest.mark.parametrize("name", ["model_dla34", "dcn_default", "decode", "jpeg"])
def test_second_device(name):
    """The case on cuda:1 while cuda:0 is current: the device guard of _lib.launch and the per-device caches (the SM
    count, the once-per-device shared-memory attribute, the decode workspace) must give cuda:0's results."""
    dev1 = torch.device("cuda:1")
    want, _ = run_leg(BUILD[name](DEV), DEV)
    with torch.cuda.device(DEV):
        case = BUILD[name](dev1)
        got, _ = run_leg(case, dev1, guard=False)
        assert torch.cuda.current_device() == 0
    same([g.to(DEV) for g in got], want, "%s on cuda:1" % name, case.loose)
    check_held(case, dev1)
