"""Cases and helpers of the training keypoint heads' tests (tests/test_heads_train_gpu.py, tests/test_heads_train_cpu.py):
the shape table, the backward's chunk and split rule restated from csrc/heads_train.cu, the inputs, the float64 / fp32
restatement computed image-chunk by image-chunk and the device call.  A helper module: it holds no tests."""
import torch
import torch.nn.functional as F

from centerpose_b200.heads_train import HEADS, OUTPUTS

DEV = torch.device("cuda:0")
PRECISIONS = ("default", "fp32")
GRAD_NAMES = ("grad_x", "grad_w0", "grad_b0", "grad_w2", "grad_b2")

# backbone -> (C, hc) of its KeypointHead
CONFIGS = {"dla_34": (64, 256), "res_50": (256, 64), "hrnet_w32": (32, 64), "hrnet_w48": (48, 64),
           "mobilenetv3": (24, 256), "mobilenetv2": (24, 256), "hardnet": (48, 256), "ghostnet": (160, 256)}
# (B, C, H, W, hc): odd shapes -- 1x1 and 7x13 maps, C = 3, hc = 8 and 40 (a partial hidden chunk), B = 1, and maps
# whose pixel count is not a multiple of the 128-pixel tile
ODD = [(1, 3, 1, 1, 8), (2, 3, 7, 13, 8), (1, 8, 7, 13, 40), (2, 70, 9, 15, 40), (3, 5, 1, 9, 16)]
# the GPU tests' shapes: integer-exact on every configuration at R = 32; accurate at R = 128 (B = 2), at the per-GPU
# batches of DLA-34's and MobileNetV3's yamls (18 and 21: 2 images per backward chunk, the last one short), at a
# 160x160 map (one image per chunk) and on the odd shapes
EXACT = [(2, C, 32, 32, hc) for C, hc in CONFIGS.values()] + ODD
ACCURACY = [(2, C, 128, 128, hc) for C, hc in CONFIGS.values()] + \
    [(18, 64, 128, 128, 256), (21, 24, 128, 128, 256), (2, 24, 160, 160, 256)] + ODD
DETERMINISM = [(2, 64, 128, 128, 256), (18, 64, 128, 128, 256)]
MEMORY = (8, 64, 128, 128, 256)
ALL_SHAPES = EXACT + ACCURACY + DETERMINISM + [MEMORY]

# the stream cases of include/centerpose_b200_heads_train.h (tests/test_heads_train_streams_gpu.py): each holds its
# call on a side stream, as tests/test_streams_gpu.py does for centerpose_b200.h, and names the entry points it reaches
STREAM_CASES = {"heads_train_default": ("heads_train_forward", "heads_train_backward"),
                "heads_train_fp32": ("heads_train_forward", "heads_train_backward")}


def shape_id(s):
    return "b%d_c%d_%dx%d_hc%d" % s


# ---- the backward's workspace (csrc/heads_train.cu make_plan, wgrad_split) ---------------------------------------
BM, BN, BK = 64, 128, 16
DH_CHUNK_BYTES = 256 << 20
TARGET_CTAS = 264
WS_CAP = 16 << 20
NOUT = sum(OUTPUTS)


def chunk_images(B, H, W, hc):
    """Images per chunk of the backward: d_hidden of all six heads for one chunk at most 256 MiB."""
    return max(1, min(B, DH_CHUNK_BYTES // (6 * hc * H * W * 4)))


def wgrad_split(nimg, C, H, W, hc):
    """(splits, K steps per split) of dW0 over the nimg * H * W pixels of a chunk."""
    K, NR = 9 * C, 6 * hc
    tiles = -(-K // BN) * -(-NR // BM)
    nsteps = -(-nimg * H * W // BK)
    s = max(1, min(-(-TARGET_CTAS // tiles), WS_CAP // (NR * K * 4), nsteps))
    steps = -(-nsteps // s)
    return -(-nsteps // steps), steps


def workspace_bytes(B, C, H, W, hc):
    n = chunk_images(B, H, W, hc)
    last = B % n or n
    splits = max(wgrad_split(n, C, H, W, hc)[0], wgrad_split(last, C, H, W, hc)[0])
    tiles = -(-H * W // BN)
    return 4 * (n * 6 * hc * H * W + n * tiles * (NOUT * hc + 6 * hc + NOUT) + splits * 6 * hc * C * 9)


# ---- inputs ------------------------------------------------------------------------------------------------------
def make_inputs(B, C, H, W, hc, seed, integer=False):
    """x, the 24 parameters in HEADS order (w0, b0, w2, b2 per head) and the six grad_outputs, on the device.
    ``integer``: integer x and grad_output in [-3, 3], weights in {-1, -1/2, 0, 1/2, 1} and biases in [-4, 4], so every
    product and sum the heads form is exact in fp32 and in the tf32 split."""
    g = torch.Generator().manual_seed(seed)
    if integer:
        def ints(shape, lo, hi, scale=1.0):
            return torch.randint(lo, hi + 1, shape, generator=g).float() * scale
        x = ints((B, C, H, W), -3, 3)
        params = []
        for c in OUTPUTS:
            params += [ints((hc, C, 3, 3), -2, 2, 0.5), ints((hc,), -4, 4), ints((c, hc, 1, 1), -2, 2, 0.5),
                       ints((c,), -4, 4)]
        gos = [ints((B, c, H, W), -3, 3) for c in OUTPUTS]
    else:
        # x, W0 and b0 on a dyadic grid (x in [0, 4) at 2^-4, W0 at 2^-6 below 1/4, b0 at 2^-10): every hidden
        # pre-activation is then exact in fp32, so the ReLU mask is float64's in every arm.  A pre-activation within
        # rounding of 0 would otherwise flip the mask in one arm and not in another, and the gradients with it, which
        # no kernel error causes.  W2, b2 and grad_output are full-precision randn, so the output and every gradient
        # are rounded as in training.
        def grid(t, step, lim):
            return (t.clamp(-lim, lim - step) / step).round() * step
        x = grid(torch.relu(torch.randn(B, C, H, W, generator=g)), 2 ** -4, 4)
        params = []
        for c in OUTPUTS:
            params += [grid(torch.randn(hc, C, 3, 3, generator=g) / (3 * C ** 0.5), 2 ** -6, 0.25),
                       grid(torch.randn(hc, generator=g) * 0.1, 2 ** -10, 1),
                       torch.randn(c, hc, 1, 1, generator=g) / hc ** 0.5, torch.randn(c, generator=g) * 0.1]
        gos = [torch.randn(B, c, H, W, generator=g) for c in OUTPUTS]
    return x.to(DEV), [p.to(DEV) for p in params], [t.to(DEV) for t in gos]


# ---- the restatement, image-chunk by image-chunk -----------------------------------------------------------------
CHUNK_BYTES = 2 << 30


def restate_chunk(B, C, H, W, hc):
    """Images per chunk of the float64 restatement: its graph (some 4 hidden maps per head) under CHUNK_BYTES."""
    return max(1, min(B, CHUNK_BYTES // (24 * hc * H * W * 8 + 8 * C * H * W * 8)))


def heads_torch(x, params):
    outs = []
    for h in range(6):
        w0, b0, w2, b2 = params[4 * h:4 * h + 4]
        outs.append(F.conv2d(F.relu(F.conv2d(x, w0, b0, padding=1)), w2, b2))
    return outs


def restated(x, params, gos, dtype, need_x=True):
    """(six outputs, grad_x, [24 parameter grads]) of torch autograd in ``dtype``; None grad_outputs leave their
    heads' parameter grads None.  Parameter grads are summed over the chunks in ``dtype``, in chunk order."""
    B, C, H, W = x.shape
    hc = params[0].shape[0]
    n = restate_chunk(B, C, H, W, hc)
    ps = [p.to(dtype) for p in params]
    outs, gxs, pgs = [], [], [None] * 24
    for b0 in range(0, B, n):
        xs = x[b0:b0 + n].to(dtype).requires_grad_(need_x)
        leaves = [p.detach().clone().requires_grad_(True) for p in ps]
        o = heads_torch(xs, leaves)
        pairs = [(t, g[b0:b0 + n].to(dtype)) for t, g in zip(o, gos) if g is not None]
        if pairs:
            torch.autograd.backward([t for t, _ in pairs], [g for _, g in pairs])
        outs.append([t.detach() for t in o])
        if need_x:
            gxs.append(xs.grad if xs.grad is not None else torch.zeros_like(xs))
        for i, l in enumerate(leaves):
            if l.grad is not None:
                pgs[i] = l.grad if pgs[i] is None else pgs[i] + l.grad
        del o, pairs, leaves
    return [torch.cat(t) for t in zip(*outs)], (torch.cat(gxs) if need_x else None), pgs


def device(x, params, gos, precision, need_x=True):
    """(six outputs, grad_x, [24 parameter grads]) of centerpose_b200.heads_train."""
    from centerpose_b200 import heads_train
    outs = heads_train.heads_forward(x, params, precision)
    gx, grads = heads_train.heads_backward(x, params, gos, need_x=need_x, precision=precision)
    return outs, gx, grads


def flat(res):
    """The outputs and every gradient as a list of (name, tensor), None entries dropped."""
    outs, gx, grads = res
    items = [("out " + h, o) for h, o in zip(HEADS, outs)]
    if gx is not None:
        items.append(("grad_x", gx))
    names = [h + "." + n for h in HEADS for n in ("w0", "b0", "w2", "b2")]
    return items + [(n, g) for n, g in zip(names, grads) if g is not None]
