"""Cases and helpers of the training DCNv2's tests (tests/test_dcn_train_gpu.py, tests/test_dcn_train_models_gpu.py,
tests/test_dcn_train_cpu.py): the shape table, the weight gradient's split-K rule restated from csrc/dcn_train.cu,
the inputs, the float64 / fp32 restatement computed image-chunk by image-chunk, the device call and the accuracy bound.
A helper module: it holds no tests."""
import math

import torch

from oracle import dcn_ref, dcn_train_ref

DEV = torch.device("cuda:0")
NAMES = ("out", "grad_input", "grad_offset", "grad_mask", "grad_weight", "grad_bias")
PRECISIONS = ("default", "fp32")
CFG = (3, 3, 1, 1, 1, 1, 1, 1, 1)

# (C, Co, H, W): every DCN of DLA-34 and MobileNetV3 at its map size for a 512x512 input, then odd shapes
DLA34 = [(512, 256, 16, 16), (256, 256, 32, 32), (256, 128, 32, 32), (128, 128, 64, 64), (128, 64, 64, 64),
         (256, 64, 32, 32), (64, 64, 128, 128)]
MOBILENETV3 = [(40, 24, 64, 64), (160, 24, 32, 32), (960, 24, 16, 16), (24, 24, 128, 128), (24, 24, 64, 64),
               (24, 24, 32, 32)]
ODD = [(8, 8, 7, 13), (8, 8, 1, 1), (64, 8, 7, 13), (8, 64, 13, 7), (3, 5, 2, 3), (24, 24, 1, 9)]
# (B, C, Co, H, W) of the accuracy test: the shapes above at B = 2; every DCN at the batch a training step runs it
# (DLA-34 at 32, MobileNetV3 at 64, as tools/bench_dcn_train.py); and 1024 -> 256 on 9x7, whose 288 output tiles give
# the weight gradient one split of several K steps
TRAINING = [(32,) + s for s in DLA34] + [(64,) + s for s in MOBILENETV3]
ACCURACY = [(2,) + s for s in DLA34 + MOBILENETV3 + ODD] + TRAINING + [(3, 1024, 256, 9, 7)]


def case_id(case):
    """The B = 2 cases keep their ids of the shape alone."""
    B, shape = case[0], case[1:]
    return ("%dx%d_%dx%d" % shape) if B == 2 else ("b%d_%dx%d_%dx%d" % case)


# ---- the weight gradient's split K (csrc/dcn_train.cu wgrad_split) ------------------------------------------------
BM, BN, BK = 64, 128, 16            # the CTA tile: Co rows, C*9 columns, pixels per K step
TARGET_CTAS = 264
WS_CAP = 16 << 20


def wgrad_split(B, C, H, W, Co):
    """(splits, K steps per split) of the weight gradient: the K = B*H*W pixels go in steps of BK to at most
    ceil(264 / output tiles) splits, capped by the 16 MiB workspace and by the number of steps."""
    K = 9 * C
    tiles = -(-K // BN) * -(-Co // BM)
    nsteps = -(-B * H * W // BK)
    s = max(1, min(-(-TARGET_CTAS // tiles), WS_CAP // (Co * K * 4), nsteps))
    steps = -(-nsteps // s)
    return -(-nsteps // steps), steps


def split_regimes(B, C, H, W, Co):
    """The regimes of wgrad_split that shape (B, C, H, W, Co) reaches."""
    splits, steps = wgrad_split(B, C, H, W, Co)
    HW, NQ = H * W, B * H * W
    nsteps = -(-NQ // BK)
    bounds = [s * steps * BK for s in range(1, splits)]
    got = set()
    if steps == 1:
        got.add("one step per split")
    if any(q // HW != (min(q + BK, NQ) - 1) // HW for q in range(0, NQ, BK)):
        got.add("step spans images")
    if nsteps - (splits - 1) * steps < steps:
        got.add("short last split")
    if any(q % HW for q in bounds):
        got.add("split boundary inside an image")
    if splits > 100:
        got.add("over 100 splits")
    if splits == 1 and steps > 1:
        got.add("one split of several steps")
    if steps > 400:
        got.add("over 400 steps per split")
    return got


REGIMES = ("one step per split", "step spans images", "short last split", "split boundary inside an image",
           "over 100 splits", "one split of several steps", "over 400 steps per split")


# ---- inputs ------------------------------------------------------------------------------------------------------
def make_inputs(B, C, Co, H, W, seed, stats="randn"):
    """The op's six inputs on the device.  ``stats``:
      * "randn": zero-mean randn input and grad_out, offsets of 2 px, uniform masks;
      * "same_sign", "sparse": training's statistics -- post-ReLU inputs, offsets at the conditioned init's scale
        (0.5 px), masks saturated near 0 and 1 (the sigmoid of 8 randn), and grad_out |randn| (every element of one
        sign) or sparse: about 1 in 1 000 entries nonzero, randn * 1e3, as the focal loss sends back from the peaks."""
    if stats not in ("randn", "same_sign", "sparse"):
        raise ValueError(stats)
    g = torch.Generator(device="cpu").manual_seed(seed)
    stdv = 1.0 / math.sqrt(9 * C)
    t = dict(input=torch.randn(B, C, H, W, generator=g), weight=(torch.rand(Co, C, 3, 3, generator=g) * 2 - 1) * stdv,
             bias=torch.randn(Co, generator=g) * 0.1, offset=torch.randn(B, 18, H, W, generator=g) * 2,
             mask=torch.rand(B, 9, H, W, generator=g), grad_out=torch.randn(B, Co, H, W, generator=g))
    if stats != "randn":
        t["input"] = torch.relu(t["input"])
        t["offset"] = t["offset"] * 0.25
        t["mask"] = torch.sigmoid(torch.randn(B, 9, H, W, generator=g) * 8)
        if stats == "same_sign":
            t["grad_out"] = t["grad_out"].abs()
        else:
            keep = torch.rand(B, Co, H, W, generator=g) < 1e-3
            t["grad_out"] = torch.where(keep, t["grad_out"] * 1e3, torch.zeros(()))
    return {k: v.to(DEV) for k, v in t.items()}


# ---- the restatement, image-chunk by image-chunk -----------------------------------------------------------------
CHUNK_BYTES = 4 << 30
GRAPH_COLUMNS = 100     # autograd through dcn_ref.dcn_v2_forward holds some 100 (C, H, W) tensors per image


def chunk_images(B, C, H, W):
    """Images per chunk of the restatement: its float64 autograd graph stays under CHUNK_BYTES.  The same in both
    dtypes, so the fp32 baseline sums the same chunks."""
    return max(1, min(B, CHUNK_BYTES // (GRAPH_COLUMNS * C * H * W * 8)))


def restated(t, dtype):
    """Output and the five gradients of autograd through the restatement, in ``dtype``.  The output, grad_input,
    grad_offset and grad_mask are per image: the chunks' are concatenated.  grad_weight and grad_bias are the sum of
    the chunks', added in ``dtype`` in chunk order."""
    B, C, H, W = t["input"].shape
    n = chunk_images(B, C, H, W)
    c = {k: v.to(dtype) for k, v in t.items()}
    per_image, gw, gb = [], None, None
    for b0 in range(0, B, n):
        s = {k: (v if k in ("weight", "bias") else v[b0:b0 + n]) for k, v in c.items()}
        out = dcn_ref.dcn_v2_forward(s["input"], s["weight"], s["bias"], s["offset"], s["mask"])
        gi, go, gm, w, b = dcn_train_ref.dcn_v2_backward(s["input"], s["weight"], s["bias"], s["offset"], s["mask"],
                                                         s["grad_out"])
        per_image.append([out.detach(), gi.detach(), go.detach(), gm.detach()])
        gw, gb = (w.detach(), b.detach()) if gw is None else (gw + w.detach(), gb + b.detach())
        del out, gi, go, gm, w, b
    return [torch.cat(p) for p in zip(*per_image)] + [gw, gb]


def device(t, precision):
    from centerpose_b200 import dcn
    out = dcn.dcn_v2_forward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], *CFG, precision=precision)
    grads = dcn.dcn_v2_backward(t["input"], t["weight"], t["bias"], t["offset"], t["mask"], t["grad_out"], *CFG,
                                precision=precision)
    return [out] + list(grads)


# ---- the bound ---------------------------------------------------------------------------------------------------
def stats(got, want):
    """(max|got - want| / max|want|, relative L2 error); absolute where ``want`` is all zero."""
    d = (got.double() - want.double()).abs()
    mx = want.abs().max().item()
    l2 = want.double().norm().item()
    return (d.max().item() / mx if mx > 0 else d.max().item(),
            (d.norm().item() / l2) if l2 > 0 else d.norm().item())


def bound_failures(label, got, ref64, ref32):
    """Each statistic of ``got`` against ``ref64`` that exceeds max(4 * e32, 1e-6), e32 being ``ref32``'s."""
    e_dev, e32 = stats(got, ref64), stats(ref32, ref64)
    return ["%s %s: %.3g > max(4 * %.3g, 1e-6)" % (label, what, a, b)
            for what, a, b in zip(("max", "l2"), e_dev, e32) if a > max(4 * b, 1e-6)]


def check_accuracy(got, ref64, ref32, label, report=None):
    """The output and five gradients ``got`` within max(4 * e32, 1e-6) of ``ref64`` on both statistics.  ``report``,
    a dict, collects {(label, name): (device's statistics, e32's)}."""
    bad = []
    for name, g, r, r32 in zip(NAMES, got, ref64, ref32):
        assert g.shape == r.shape and g.dtype == torch.float32, name
        assert torch.isfinite(g).all(), "%s %s: not finite" % (label, name)
        if report is not None:
            report[(label, name)] = (stats(g, r), stats(r32, r))
        bad += bound_failures("%s %s" % (label, name), g, r, r32)
    assert not bad, "\n".join(bad)
