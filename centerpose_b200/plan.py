"""Graph builder: lowers a backbone + head description to a flat program of fused CUDA ops
(``cpb200_op``, ``include/centerpose_b200.h``) and owns the device buffers it runs on.

What gets fused at lowering time (reference modules in brackets):
  * eval-mode ``BatchNorm2d`` folded into the preceding conv / DCN weights and bias
    (``pose_dla_dcn.py:43-57,155-163,199-204,336-348``; eps 1e-5);
  * ReLU and residual add run in the conv epilogue (``BasicBlock.forward``);
  * ``Root``'s ``torch.cat`` is never materialised: each child is one K-slab input of the 1x1
    conv (``pose_dla_dcn.py:155-163``);
  * IDAUp's depthwise ``ConvTranspose2d`` + ``layers[i] + layers[i-1]`` is one op
    (``pose_dla_dcn.py:371-377``);
  * DCN: offset/mask conv -> one op; sigmoid(mask) * bilinear gather * GEMM + BN + ReLU ->
    one op (``DCNv2/dcn_v2.py:117-127``), no ``columns`` scratch in HBM.

All torch usage here is plumbing (device memory, one-time weight re-layout).
"""
from __future__ import annotations

import ctypes
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib

OP_CONV, OP_STEM, OP_MAXPOOL, OP_DWDECONV_ADD, OP_DCN, OP_UPSAMPLE_ADD = 1, 2, 3, 4, 5, 7      # 6 is retired
OP_DWCONV, OP_AVGPOOL, OP_SCALE_ADD, OP_CONVERT, OP_S2D = 8, 9, 10, 11, 12
OP_AVGPOOL2, OP_RESIZE_BILINEAR, OP_HEADS = 13, 14, 15
FLAG_RELU, FLAG_OUT_NCHW_F32, FLAG_OUT_F32, FLAG_TC, FLAG_HSWISH, FLAG_HSIGMOID, FLAG_TO_F32 = 1, 2, 4, 8, 16, 32, 64
FLAG_RELU6, FLAG_CLIP01 = 128, 256
_ACT_FLAG = {None: 0, "relu": FLAG_RELU, "hswish": FLAG_HSWISH, "hsigmoid": FLAG_HSIGMOID, "relu6": FLAG_RELU6,
             "clip01": FLAG_CLIP01}
F32, BF16, BF16X2, F16X2 = 0, 1, 2, 3
PRECISIONS = {"fp32": F32, "bf16": BF16, "bf16x2": BF16X2, "fp16x2": F16X2}
BN_EPS = 1e-5


# The wgmma fp32 accumulator rounds TOWARD ZERO at every instruction.  For dot products of random-sign operands this
# shrinks the result by a factor that is linear in the number of K = 16 accumulation steps — measured on an H100 SXM
# (400 W power limit) with iid Gaussian and post-ReLU operands (CPB200_RZ_COMP=0 python tools/rz_probe.py): -1.6e-8 per
# step with fp16 planes (K = 256 .. 4608), -1.0e-8 .. -1.5e-8 with bf16 planes.  Uncorrected it is the dominant error of
# the split precisions through a deep network because it is COHERENT: it adds up over the ~40 layers of DLA-34 and the
# chained DCNs amplify it towards the heads (tools/layer_err.py shows it per layer).  The host therefore folds the expected
# factor 1 + beta * K/16 into cpb200_op.acc_scale (a multiplication the epilogue performs anyway).  CPB200_RZ_COMP
# overrides beta (0 disables); all-positive dot products shrink ~6x more and stay under-corrected.
RZ_BETA = {"fp16x2": 1.6e-8, "bf16x2": 1.2e-8}


def rz_compensation(precision: str, k_total: int) -> float:
    e = os.environ.get("CPB200_RZ_COMP")
    beta = float(e) if e is not None else RZ_BETA.get(precision, 0.0)
    return 1.0 + beta * (k_total / 16.0)


def split_planes(t: torch.Tensor, dt: torch.dtype) -> torch.Tensor:
    """fp32 tensor -> (2, ...) stack of 16-bit planes: hi = rn16(t), lo = rn16(t - hi)   (include/centerpose_b200.h)."""
    t = t.float()
    if dt == torch.float16:
        t = t.clamp(-65504.0, 65504.0)
    hi = t.to(dt)
    lo = (t - hi.float()).to(dt)
    return torch.stack([hi, lo]).contiguous()


def pow2_scale(w: torch.Tensor, target_exp: int = 12) -> float:
    """Power-of-two factor that moves max|w| into [2^target_exp, 2^(target_exp+1)): applied to the weights of fp16-plane
    ops so that the lo parts are normal fp16 numbers; the kernels multiply the accumulator by its inverse (exact)."""
    m = float(w.abs().max())
    if not (m > 0.0) or m != m or m == float("inf"):
        return 1.0
    import math
    return float(2.0 ** (target_exp - math.floor(math.log2(m))))


class OpStruct(ctypes.Structure):
    _fields_ = [
        ("type", ctypes.c_int32), ("flags", ctypes.c_uint32), ("act_dtype", ctypes.c_int32),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
        ("Ho", ctypes.c_int32), ("Wo", ctypes.c_int32), ("nsrc", ctypes.c_int32),
        ("cin", ctypes.c_int32 * 4), ("cout", ctypes.c_int32),
        ("kh", ctypes.c_int32), ("kw", ctypes.c_int32), ("stride", ctypes.c_int32),
        ("pad_h", ctypes.c_int32), ("pad_w", ctypes.c_int32),
        ("out_ch_off", ctypes.c_int32), ("out_ch_total", ctypes.c_int32),
        ("Hd", ctypes.c_int32), ("Wd", ctypes.c_int32),
        ("out_sy", ctypes.c_int32), ("out_sx", ctypes.c_int32),
        ("out_oy", ctypes.c_int32), ("out_ox", ctypes.c_int32),
        ("aux_pitch", ctypes.c_int32),
        ("src", ctypes.c_void_p * 4), ("res", ctypes.c_void_p), ("aux", ctypes.c_void_p),
        ("dst", ctypes.c_void_p), ("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p),
        ("tc", ctypes.c_void_p), ("src_pitch", ctypes.c_int32 * 4),
        ("acc_scale", ctypes.c_float), ("reserved_", ctypes.c_int32),
    ]


class HeadStruct(ctypes.Structure):
    """``cpb200_head``: one entry of an OP_HEADS op's table."""
    _fields_ = [
        ("hidden", ctypes.c_int32), ("cout", ctypes.c_int32), ("weight", ctypes.c_void_p), ("bias", ctypes.c_void_p),
        ("acc_scale3", ctypes.c_float), ("acc_scale1", ctypes.c_float), ("dst", ctypes.c_void_p),
    ]


class Sym:
    """Symbolic activation tensor (NHWC unless kind says otherwise)."""
    __slots__ = ("C", "H", "W", "kind", "name", "_buf", "fixed", "parent", "ch_off", "_f32", "_sp", "keep")

    def __init__(self, C, H, W, kind="act", name="", parent=None, ch_off=0):
        self.C, self.H, self.W, self.kind, self.name = C, H, W, kind, name
        self._buf = None         # torch tensor once allocated
        self.fixed = False       # externally provided storage (network input / outputs)
        self.parent = parent     # channel slice [ch_off, ch_off + C) of `parent` (shares its storage)
        self.ch_off = ch_off
        self._f32 = None         # split precisions: cached fp32 copy / split copy of this activation
        self._sp = None
        self.keep = False        # PlanBuilder.keep_result(): never pruned, buffer never recycled (tests / diagnostics read it)

    # a slice lives in its parent's buffer and keeps the parent alive (liveness is tracked on Plan._root)
    @property
    def buf(self):
        return self.parent.buf if self.parent is not None else self._buf

    @buf.setter
    def buf(self, v):
        self._buf = v

    @property
    def pitch(self):
        return self.parent.C if self.parent is not None else self.C


@dataclass(eq=False)
class Op:
    """One op of the program, over symbolic tensors; ``Plan`` turns it into a ``cpb200_op``.  ``res`` and ``aux`` fill
    the header's fields of those names: CONV's residual is ``res``; SCALE_ADD's gate is ``res`` and its skip ``aux``;
    DCN's offset/mask tensor and the DWDECONV_ADD / UPSAMPLE_ADD skip are ``aux``.  ``out_map`` = (Hd, Wd, sy, sx, oy,
    ox) and ``HoWo`` place the result in ``dst``; by default it fills all of ``dst``."""
    type: int
    dtype: int                                   # cpb200_op.act_dtype
    srcs: List[Sym]
    dst: Sym
    cout: int
    flags: int = 0
    k: Tuple[int, int] = (1, 1)
    stride: int = 1
    pad: Tuple[int, int] = (0, 0)
    weight: Optional[torch.Tensor] = None
    bias: Optional[torch.Tensor] = None
    res: Optional[Sym] = None
    aux: Optional[Sym] = None
    aux_pitch: int = 0
    acc_scale: float = 1.0
    out_ch_off: int = 0
    out_map: Optional[Tuple[int, int, int, int, int, int]] = None
    HoWo: Optional[Tuple[int, int]] = None
    w_raw: Optional[torch.Tensor] = None         # the unpacked (Co, Ci, kh, kw) weight of a conv / DCN
    heads: Optional[List[Tuple["Op", "Op"]]] = None      # OP_HEADS: the (3x3, 1x1) conv pairs it replaces

    def __post_init__(self):
        if self.out_map is None:
            self.out_map = (self.dst.H, self.dst.W, 1, 1, 0, 0)
        if self.HoWo is None:
            self.HoWo = (self.dst.H, self.dst.W)

    def operands(self) -> List[Sym]:
        """every activation the op reads"""
        return [*self.srcs, *(s for s in (self.res, self.aux) if s is not None)]


def _swizzle_chunks(blk: torch.Tensor, key: torch.Tensor) -> torch.Tensor:
    """blk [..., row n, 16-byte chunk j, element] -> the same rows with chunk j stored at chunk j ^ key[n]: the
    shared-memory swizzles of the tensor-core stems' B operand (csrc/net_stem_tc.cu)"""
    j = torch.arange(blk.shape[-2], device=blk.device)
    idx = (j.view(1, -1, 1) ^ key.view(-1, 1, 1)).expand(blk.shape)
    return torch.zeros(blk.shape, dtype=blk.dtype, device=blk.device).scatter_(-2, idx, blk.contiguous())


def fold_bn(w: torch.Tensor, b: Optional[torch.Tensor], bn: Optional[dict], eps: float = BN_EPS):
    """conv weight (Co,Ci,kh,kw) [+bias] followed by eval BatchNorm (epsilon ``eps``) -> equivalent weight/bias."""
    w = w.float()
    co = w.shape[0]
    b = torch.zeros(co, device=w.device) if b is None else b.float()
    if bn is None:
        return w, b
    scale = bn["weight"].float() / torch.sqrt(bn["running_var"].float() + eps)
    return w * scale.view(-1, 1, 1, 1), (b - bn["running_mean"].float()) * scale + bn["bias"].float()


class PlanBuilder:
    def __init__(self, B: int, H: int, W: int, precision: str, device: torch.device, tc: Optional[bool] = None):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        self.B, self.H, self.W = B, H, W
        self.device = device
        self.precision = precision
        self.act_dtype = PRECISIONS[precision]
        # split-operand precisions: activations are hi/lo 16-bit planes, every conv runs on wgmma as three products
        self.split = precision in ("bf16x2", "fp16x2")
        self.torch16 = torch.float16 if precision == "fp16x2" else torch.bfloat16
        self.torch_act = torch.float32 if precision == "fp32" else self.torch16
        self.ops: List[Op] = []
        self.keep: List[torch.Tensor] = []      # weights / biases kept alive
        self.syms: List[Sym] = []
        # tensor-core (wgmma) path: 16-bit operands only; tc=False forces the SIMT kernels (bf16: debugging)
        if tc is None:
            tc = True
        if self.split and not tc:
            raise ValueError("split precisions run on the tensor-core path only")
        self.use_tc = bool(tc) and precision != "fp32"

    # ---- symbolic tensors -------------------------------------------------------------
    def _sym(self, C, H, W, kind="act", name=""):
        # An input too small for the network's deepest stride (HarDNet at 32 pixels: its sixth halving leaves 0 rows)
        # would lower to ops of zero extent; refuse it here, before anything is launched, as the reference's pool raises.
        if C <= 0 or H <= 0 or W <= 0:
            raise ValueError(f"centerpose_b200: a {self.H}x{self.W} input is too small for this network "
                             f"(an intermediate map would be {C}x{H}x{W})")
        s = Sym(C, H, W, kind, name)
        self.syms.append(s)
        return s

    def input(self, C=3):
        s = self._sym(C, self.H, self.W, "nchw_in", "input")
        s.fixed = True
        return s

    def external(self, t: torch.Tensor, kind="act"):
        """Wrap an existing NHWC device tensor (B,H,W,C) as a program input (tests, partial graphs).  Split
        precisions: ``t`` is fp32 and is split into the hi / lo planes here."""
        B, H, W, C = t.shape
        assert B == self.B and t.is_contiguous()
        s = self._sym(C, H, W, kind, "external")
        s.fixed = True
        s.buf = split_planes(t, self.torch16) if (self.split and kind == "act") else t
        return s

    def keep_result(self, s: Sym) -> Sym:
        """mark an intermediate as a program result: its producer is not pruned and its buffer is not recycled."""
        Plan._root(s).keep = True
        return s

    def output(self, C, H, W, name):
        s = self._sym(C, H, W, "nchw_out", name)
        s.fixed = True
        return s

    # ---- split precisions: fp32 islands for ops without a native split kernel ------------------
    def _to_f32(self, x: Optional[Sym]) -> Optional[Sym]:
        """fp32 NHWC copy of a split activation (cached; a channel slice converts its parent once)."""
        if x is None or not self.split or x.kind != "act":
            return x
        if x.parent is not None:
            return Sym(x.C, x.H, x.W, "actf32", parent=self._to_f32(x.parent), ch_off=x.ch_off)
        if x._f32 is None:
            y = self._sym(x.C, x.H, x.W, "actf32", x.name + ".f32")
            self.ops.append(Op(OP_CONVERT, self.act_dtype, [x], y, x.C, flags=FLAG_TO_F32))
            x._f32 = y; y._sp = x
        return x._f32

    def _to_split(self, y: Sym) -> Sym:
        """split copy of an fp32 NHWC activation produced inside an fp32 island."""
        if not self.split or y.kind != "actf32":
            return y
        if y._sp is None:
            x = self._sym(y.C, y.H, y.W, "act", y.name + ".sp")
            self.ops.append(Op(OP_CONVERT, self.act_dtype, [y], x, y.C))
            y._sp = x; x._f32 = y
        return y._sp

    def _island_sym(self, C, H, W):
        """output of an op that runs on fp32 in split mode (kind 'actf32'), an ordinary activation otherwise."""
        return self._sym(C, H, W, "actf32" if self.split else "act")

    def _storage(self, kind: str) -> Tuple[int, int, torch.dtype]:
        """How a tensor of this kind is stored: (bytes per NHWC element slot, bytes per element inside one plane, torch
        dtype of a plane).  Split activations are two 16-bit planes, hi then lo."""
        if kind in ("f32", "actf32") or self.act_dtype == F32:
            return 4, 4, torch.float32
        if kind != "act":
            raise KeyError(kind)
        return (4, 2, self.torch16) if self.split else (2, 2, torch.bfloat16)

    def _dev(self, t: torch.Tensor, dtype=torch.float32):
        t = t.detach().to(device=self.device, dtype=dtype).contiguous()
        self.keep.append(t)
        return t

    # ---- weight packing ------------------------------------------------------------------
    def _pack_conv(self, w: torch.Tensor):
        """(Co,Ci,kh,kw) fp32 -> SIMT layout [kh*kw][Ci][Co_pad4] fp32."""
        co, ci, kh, kw = w.shape
        cop = (co + 3) // 4 * 4
        p = torch.zeros(kh * kw, ci, cop, dtype=torch.float32, device=w.device)
        p[:, :, :co] = w.permute(2, 3, 1, 0).reshape(kh * kw, ci, co)
        return self._dev(p)

    def _pack_conv_tc(self, w: torch.Tensor, bk: int) -> Tuple[torch.Tensor, float]:
        """(Co,Ci,kh,kw) fp32 -> wgmma layout [kh*kw][Ci/bk][Co_pad16][bk] bf16 (K-major B operand, slab-major:
        the rows of one (tap, K-slab) block are contiguous, so a TMA weight box is one dense run of memory instead of
        Co rows strided by Ci), and the factor the weights were multiplied by.  bk = the kernels' K-slab width."""
        co, ci, kh, kw = w.shape
        assert ci % bk == 0
        cop = (co + 15) // 16 * 16
        p = torch.zeros(kh * kw, ci // bk, cop, bk, dtype=torch.float32, device=w.device)
        p[:, :, :co, :] = w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci // bk, bk).permute(0, 2, 1, 3)
        if self.split:
            # [plane][tap][slab][Co_pad][bk]: hi plane then lo plane; fp16 planes carry the weights times a power of two
            # (pow2_scale) whose inverse the kernel applies to the accumulator (cpb200_op.acc_scale)
            scale = pow2_scale(w) if self.torch16 == torch.float16 else 1.0
            return self._dev(split_planes(p * scale, self.torch16), self.torch16), scale
        return self._dev(p, torch.bfloat16), 1.0

    def _acc_scale(self, k_total: int, scale: float) -> float:
        """cpb200_op.acc_scale of a tensor-core op that sums k_total products over weights packed times ``scale``: split
        precisions undo the scale and compensate the accumulator's rounding toward zero (rz_compensation)."""
        return rz_compensation(self.precision, k_total) / scale if self.split else 1.0

    @staticmethod
    def _tc_bk(srcs) -> int:
        """K-slab width the tensor-core kernels use for these inputs (64 / 32 / 16): mirrors tc::slab_for (csrc/net_tc.cu)."""
        bk = 64
        for s in srcs:
            if s.C % 64:
                bk = min(bk, 32 if s.C % 32 == 0 else 16)
        return bk

    def channel_slice(self, x: Sym, off: int, c: int) -> Sym:
        """View of channels [off, off+c) of an NHWC activation (no copy): readable by conv ops through the op's
        ``src_pitch`` field.  Used to feed the six head 1x1 convs from ONE fused hidden tensor."""
        assert x.parent is None and x.kind == "act" and 0 <= off and off + c <= x.C and off % 16 == 0 and c % 16 == 0
        return Sym(c, x.H, x.W, "act", parent=x, ch_off=off)

    def _pack_stem_tc(self, w: torch.Tensor):
        """(N,3,7,7) fp32 -> the 128-byte-swizzled K-major B operand image of csrc/net_stem_tc.cu:
        k = (c*7 + r)*8 + s (s = 7 and k >= 168 are zero), three 64-wide slabs of N rows x 128 bytes,
        16-byte chunk j of row n stored at chunk j ^ (n & 7)."""
        N = w.shape[0]
        wk = torch.zeros(N, 3, 7, 8, dtype=torch.float32, device=w.device)
        wk[..., :7] = w.float()
        wk = torch.nn.functional.pad(wk.reshape(N, 168), (0, 24))                   # (N, 192)
        blk = wk.reshape(N, 3, 8, 8).permute(1, 0, 2, 3)                            # [slab][n][chunk j][e]
        return self._dev(_swizzle_chunks(blk, torch.arange(N, device=w.device) & 7), torch.bfloat16)

    def _pack_stem_tc_h(self, w: torch.Tensor) -> Tuple[torch.Tensor, float]:
        """(N,3,7,7) fp32 -> B operand image of the stride-1 tensor-core stem (stem_tc_h_kernel): one block per
        horizontal tap s of N rows x 64 bytes, k = c*7 + r (21 real of 32), 64-byte swizzle: 16-byte chunk j of
        row n stored at chunk j ^ ((n >> 1) & 3) (tap blocks are multiples of 1024 bytes); and the factor the weights
        were multiplied by."""
        N = w.shape[0]
        wk = torch.zeros(7, N, 32, dtype=torch.float32, device=w.device)                # [s][n][k]
        wk[:, :, :21] = w.float().permute(3, 0, 1, 2).reshape(7, N, 21)
        blk = wk.reshape(7, N, 4, 8)                                                     # [s][n][chunk j][e]
        key = (torch.arange(N, device=w.device) >> 1) & 3
        if self.split:
            # per tap [hi tile (N rows) | lo tile (N rows)]; row n' = plane * N + n of the 2N-row block is swizzled with
            # (n' >> 1) & 3 == (n >> 1) & 3 (N is a multiple of 8)
            scale = pow2_scale(w) if self.torch16 == torch.float16 else 1.0
            planes = split_planes(blk * scale, self.torch16)                             # (2, 7, N, 4, 8)
            return self._dev(_swizzle_chunks(planes, key).transpose(0, 1).contiguous(), self.torch16), scale
        return self._dev(_swizzle_chunks(blk, key), torch.bfloat16), 1.0

    def _tc_ok(self, srcs, co, kh, kw, stride, out, out_map, Wo):
        return (self.use_tc and stride in (1, 2) and Wo >= 8
                and all(s.C % 16 == 0 and s.kind == "act" for s in srcs)
                and (co % 16 == 0 or out in ("f32", "nchw")) and kh * kw <= 49)

    # ---- ops -------------------------------------------------------------------------------
    # Split precisions (bf16x2 / fp16x2): convs, DCNs and the stride-1 stem run natively on the hi/lo planes (tensor-core
    # kernels), and so do the element-wise ops (_eltwise); everything else (conv shapes the tensor-core kernels do not
    # take, e.g. maps narrower than 8 pixels, and element-wise ops on channel slices) runs on fp32 between two CONVERT
    # ops — an "fp32 island": slower, never less precise.
    def stem(self, x: Sym, w, b, k, stride, pad, relu=True, act=None):
        co, ci = w.shape[0], w.shape[1]
        if (self.use_tc and self.split and stride == 2 and ci == 3 and k in (3, 7) and pad == k // 2
                and co % 16 == 0 and x.H % 2 == 0 and x.W % 2 == 0 and x.kind == "nchw_in"
                and os.environ.get("CPB200_S2D_STEM", "1") != "0"):
            # Stride-2 stems in split precisions (ResNet 7x7, HRNet 3x3): space-to-depth of the image (OP_S2D: 2x2 pixel
            # blocks -> 12 of 16 channels) turns  out[o] = sum_r w[r] x[2o - pad + r]  into a STRIDE-1 conv over the half-
            # resolution map: input index 2o - pad + r = 2 (o + q) + parity with q = floor((r - pad) / 2), parity =
            # (r - pad) & 1, so a 7-tap filter becomes taps q = -2..1 (a 5x5 conv, pad 2, last tap zero) and a 3-tap filter
            # q = -1..0 (a 3x3 conv, pad 1).  It then runs on the split tensor-core halo kernel instead of a CUDA-core
            # fp32 island (ResNet-50 B=16: 954 us + a CONVERT pass).
            z = self._sym(16, x.H // 2, x.W // 2)
            self.ops.append(Op(OP_S2D, self.act_dtype, [x], z, 16, k=(2, 2), stride=2))
            k2 = (k + 1) // 2 + 1
            p2 = k2 // 2
            w2 = torch.zeros(co, 16, k2, k2, dtype=torch.float32, device=w.device)
            wf = w.float()
            for r in range(k):
                qy, py = (r - pad) // 2, (r - pad) & 1
                for q in range(k):
                    qx, px = (q - pad) // 2, (q - pad) & 1
                    c0 = (py * 2 + px) * 3
                    w2[:, c0:c0 + 3, qy + p2, qx + p2] = wf[:, :, r, q]
            return self.conv([z], w2, b.float(), stride=1, pad=p2, relu=relu, act=act)
        flags = _ACT_FLAG[act] if act else (FLAG_RELU if relu else 0)
        Ho = (x.H + 2 * pad - k) // stride + 1; Wo = (x.W + 2 * pad - k) // stride + 1
        if (self.use_tc and k == 7 and ci == 3 and pad == 3 and stride in (1, 2) and co in (16, 64)
                and not (self.split and stride != 1)):
            # tensor-core stem with the im2col done in shared memory (csrc/net_stem_tc.cu); split precisions: stride 1 only
            y = self._sym(co, Ho, Wo)
            wp, scale = self._pack_stem_tc_h(w) if stride == 1 else (self._pack_stem_tc(w), 1.0)
            self.ops.append(Op(OP_STEM, self.act_dtype, [x], y, co, flags=flags | FLAG_TC, k=(k, k), stride=stride,
                               pad=(pad, pad), weight=wp, bias=self._dev(b), acc_scale=self._acc_scale(7 * 32, scale)))
            return y
        y = self._island_sym(co, Ho, Wo)
        wp = self._dev(w.permute(2, 3, 1, 0).reshape(k * k * ci, co))
        self.ops.append(Op(OP_STEM, F32 if self.split else self.act_dtype, [x], y, co, flags=flags, k=(k, k),
                           stride=stride, pad=(pad, pad), weight=wp, bias=self._dev(b)))
        return self._to_split(y)

    def conv(self, srcs: Sequence[Sym], w, b, stride=1, pad=0, relu=False, res: Optional[Sym] = None,
             out: str = "act", dst: Optional[Sym] = None, ch_off: int = 0, pad_hw=None,
             out_map=None, act=None, _island_dst: Optional[Sym] = None):
        """w (Co, sum(Ci), kh, kw) already BN-folded; b (Co).  out: 'act' | 'f32' | 'nchw'.
        pad_hw=(top,left) overrides symmetric padding; out_map=(Hd,Wd,sy,sx,oy,ox,Ho,Wo) writes a
        strided sub-lattice of a larger dst (used to lower dense ConvTranspose2d)."""
        co, ci, kh, kw = w.shape
        assert ci == sum(s.C for s in srcs), (ci, [s.C for s in srcs])
        H, W = srcs[0].H, srcs[0].W
        ph, pw = pad_hw if pad_hw is not None else (pad, pad)
        if out_map is None:
            Ho = (H + 2 * ph - kh) // stride + 1; Wo = (W + 2 * pw - kw) // stride + 1
            Hd, Wd, sy, sx, oy, ox = Ho, Wo, 1, 1, 0, 0
        else:
            Hd, Wd, sy, sx, oy, ox, Ho, Wo = out_map
        flags = _ACT_FLAG[act] if act else (FLAG_RELU if relu else 0)     # act: a key of _ACT_FLAG
        tc = self._tc_ok(srcs, co, kh, kw, stride, out, out_map, Wo)
        island = self.split and not tc                                     # fp32 island (see above)
        if island:
            srcs = [self._to_f32(s_) for s_ in srcs]
            res = self._to_f32(res)
        if out == "nchw":
            assert dst is not None
            flags |= FLAG_OUT_NCHW_F32
            y = dst
        elif out == "f32":
            flags |= FLAG_OUT_F32
            y = dst if dst is not None else self._sym(co, Hd, Wd, "f32")
        elif island:
            assert dst is None, "strided-output convs go through deconv_k4s2"
            y = _island_dst if _island_dst is not None else self._sym(co, Hd, Wd, "actf32")
        else:
            y = dst if dst is not None else self._sym(co, Hd, Wd)
        if tc:
            flags |= FLAG_TC
            wp, scale = self._pack_conv_tc(w, self._tc_bk(srcs))
            acc_scale = self._acc_scale(kh * kw * ci, scale)
        else:
            wp, acc_scale = self._pack_conv(w), 1.0
        self.ops.append(Op(OP_CONV, F32 if island else self.act_dtype, list(srcs), y, co, flags=flags, k=(kh, kw),
                           stride=stride, pad=(ph, pw), weight=wp, bias=self._dev(b), res=res, acc_scale=acc_scale,
                           out_ch_off=ch_off, out_map=(Hd, Wd, sy, sx, oy, ox), HoWo=(Ho, Wo), w_raw=w))
        if island and out == "act" and _island_dst is None:
            return self._to_split(y)
        return y

    _KSEL = {0: [3, 1], 1: [2, 0]}        # kernel rows/cols feeding output parity 0 / 1, in input order

    def deconv_k4s2(self, x: Sym, w_full, b, relu=True) -> Sym:
        """Dense ConvTranspose2d(k4, s2, p1) (msra_resnet.py:168-193) as four 2x2 parity convs writing the strided
        sub-lattices of one output tensor.  w_full (Cout, Cin, 4, 4) BN-folded."""
        co = w_full.shape[0]
        Ho, Wo = 2 * x.H, 2 * x.W
        tc = self._tc_ok([x], co, 2, 2, 1, "act", (Ho, Wo, 2, 2, 0, 0, x.H, x.W), x.W)
        island = self.split and not tc
        y = self._sym(co, Ho, Wo, "actf32" if island else "act")
        for a in (0, 1):
            for bb in (0, 1):
                w_sub = w_full[:, :, self._KSEL[a], :][:, :, :, self._KSEL[bb]].contiguous()        # (Cout, Cin, 2, 2)
                self.conv([x], w_sub, b, stride=1, relu=relu, dst=None if island else y, _island_dst=y if island else None,
                          pad_hw=(1 - a, 1 - bb), out_map=(Ho, Wo, 2, 2, a, bb, x.H, x.W))
        return self._to_split(y) if island else y

    def _eltwise(self, op_type: int, x: Sym, C, H, W, aux: Optional[Sym] = None, gate: Optional[Sym] = None,
                 f32_out=False, **fields) -> Sym:
        """Emit an element-wise op (csrc/net_simt.cu: run_eltwise) of C output channels; ``fields`` are the rest of its
        Op.  fp32 / bf16 run it natively.  Split precisions run it on the planes (SpC / SpM handles) when every
        activation operand is a whole split tensor; there the SCALE_ADD ``gate`` (the op's ``res``) is read as fp32 and
        ``f32_out`` (AVGPOOL) writes an fp32 result.  Otherwise it runs on fp32 between CONVERT ops (an fp32 island)."""
        if self.split and all(s is None or (s.kind == "act" and s.parent is None) for s in (x, aux)) \
                and (gate is None or gate.parent is None):
            y = self._sym(C, H, W, "actf32" if f32_out else "act")
            self.ops.append(Op(op_type, self.act_dtype, [x], y, C, res=self._to_f32(gate), aux=aux, **fields))
            return self._to_split(y)
        y = self._island_sym(C, H, W)
        self.ops.append(Op(op_type, F32 if self.split else self.act_dtype, [self._to_f32(x)], y, C,
                           res=self._to_f32(gate), aux=self._to_f32(aux), **fields))
        return self._to_split(y)

    def maxpool(self, x: Sym, k=2, stride=2, pad=0):
        Ho = (x.H + 2 * pad - k) // stride + 1; Wo = (x.W + 2 * pad - k) // stride + 1
        return self._eltwise(OP_MAXPOOL, x, x.C, Ho, Wo, k=(k, k), stride=stride, pad=(pad, pad))

    def up_add(self, x: Sym, skip: Optional[Sym], w, *, b=None, act=None, stride=None, pad=None):
        """depthwise ConvTranspose2d weight (C,1,2f,2f), stride f, pad f//2, + skip.
        With a BN-folded bias ``b`` (C): act(deconv + b) + skip, and ``stride`` / ``pad`` may be given (MobileNetV2's
        IDAUp: k 2, stride 2, pad 0, ReLU, mobilenetv2.py:162-183).  Without one, ``act`` must be None."""
        C, _, k, _ = w.shape
        f = k // 2 if stride is None else stride
        p = f // 2 if pad is None else pad
        assert b is not None or act is None, "an activation needs the bias form"
        Ho = (x.H - 1) * f - 2 * p + k; Wo = (x.W - 1) * f - 2 * p + k
        wp = self._dev(w.float().reshape(C, k * k).t())          # [k*k][C]
        return self._eltwise(OP_DWDECONV_ADD, x, C, Ho, Wo, aux=skip, aux_pitch=skip.C if skip is not None else 0,
                             flags=_ACT_FLAG[act], k=(k, k), stride=f, pad=(p, p), weight=wp,
                             bias=None if b is None else self._dev(b))

    def dwconv(self, x: Sym, w, b, stride=1, act=None):
        """depthwise conv, w (C,1,k,k) BN-folded, pad k//2   (mobilenetv3.py:124-127)."""
        C, _, k, _ = w.shape
        assert C == x.C
        Ho = (x.H + 2 * (k // 2) - k) // stride + 1; Wo = (x.W + 2 * (k // 2) - k) // stride + 1
        wp = self._dev(w.float().reshape(C, k * k).t())          # [k*k][C]
        return self._eltwise(OP_DWCONV, x, C, Ho, Wo, flags=_ACT_FLAG[act], k=(k, k), stride=stride,
                             pad=(k // 2, k // 2), weight=wp, bias=self._dev(b))

    def avgpool(self, x: Sym):
        """global average pool -> (C, 1, 1)   (mobilenetv3.py:100).  Split mode: planes in, fp32 out (the 1x1-map SE convs
        that follow run on fp32 anyway)."""
        return self._eltwise(OP_AVGPOOL, x, x.C, 1, 1, f32_out=True, k=(x.H, x.W))

    def scale_add(self, x: Sym, gate: Sym, skip: Optional[Sym] = None):
        """x * gate[b, c] (+ skip)   (mobilenetv3.py:111,146).  Split mode: x / skip / result are planes, the gate is fp32."""
        assert gate.C == x.C and gate.H == 1 and gate.W == 1
        return self._eltwise(OP_SCALE_ADD, x, x.C, x.H, x.W, aux=skip, gate=gate)

    def upsample_add(self, x: Sym, skip: Optional[Sym], f: int, relu=False):
        """nearest-neighbour upsample x f of ``x`` (+ skip)(+ReLU)   (pose_higher_hrnet.py:186-187,224-232)."""
        return self._eltwise(OP_UPSAMPLE_ADD, x, x.C, x.H * f, x.W * f, aux=skip,
                             aux_pitch=skip.C if skip is not None else 0, flags=FLAG_RELU if relu else 0, stride=f)

    def avgpool2(self, x: Sym):
        """2x2 / stride-2 average pool, floor mode   (hardnet.py:141 nn.AvgPool2d(2, 2))."""
        return self._eltwise(OP_AVGPOOL2, x, x.C, x.H // 2, x.W // 2, k=(2, 2), stride=2)

    def resize_bilinear(self, x: Sym, Ho: int, Wo: int):
        """bilinear resize to (Ho, Wo) with align_corners=True   (hardnet.py:95-100, TransitionUp)."""
        return self._eltwise(OP_RESIZE_BILINEAR, x, x.C, Ho, Wo)

    def dcn(self, x: Sym, w, b, om_w, om_b, relu=True):
        """DCN module (dcn_v2.py:117-127) with BN already folded into (w, b)."""
        # offset/mask conv: 27 channels padded to 32 so every pixel row is 128 bytes (vector stores / loads)
        om_w32 = torch.zeros(32, *om_w.shape[1:], dtype=torch.float32, device=om_w.device); om_w32[:27] = om_w.float()
        om_b32 = torch.zeros(32, dtype=torch.float32, device=om_b.device); om_b32[:27] = om_b.float()
        om = self.conv([x], om_w32, om_b32, stride=1, pad=1, relu=False, out="f32")
        co = w.shape[0]
        tc = self.use_tc and x.kind == "act" and x.C % 64 == 0 and co % 16 == 0 and 32 <= co and x.W >= 8
        island = self.split and not tc
        xin = self._to_f32(x) if island else x
        y = self._sym(co, x.H, x.W, "actf32" if island else "act")
        if tc:
            wp, scale = self._pack_conv_tc(w, 64)
            acc_scale = self._acc_scale(9 * x.C, scale)
        else:
            wp, acc_scale = self._pack_conv(w), 1.0
        self.ops.append(Op(OP_DCN, F32 if island else self.act_dtype, [xin], y, co,
                           flags=(FLAG_RELU if relu else 0) | (FLAG_TC if tc else 0), k=(3, 3), pad=(1, 1), weight=wp,
                           bias=self._dev(b), aux=om, aux_pitch=om.C, acc_scale=acc_scale, w_raw=w))
        return self._to_split(y) if island else y

    # ---- finalisation -----------------------------------------------------------------------
    def build(self) -> "Plan":
        return Plan(self)


class Plan:
    """Allocated, ready-to-run op program for one (B, H, W, precision)."""

    def __init__(self, pb: PlanBuilder):
        self.pb = pb
        self.device = pb.device
        self._prune(pb)
        self._fuse_heads(pb)
        self._allocate(pb)
        n = len(pb.ops)
        self.ops = (OpStruct * n)()
        self.in_slots = []      # (op index, src slot) fed by the network input
        self.out_slots = {}     # output name -> op indices writing it, or (op index, head) of an OP_HEADS table
        self._head_tables = {}  # op index -> its cpb200_head table (host memory the op's aux points to)
        for i, po in enumerate(pb.ops):
            o = self.ops[i]
            o.type = po.type; o.flags = po.flags; o.act_dtype = po.dtype
            o.acc_scale = po.acc_scale
            s0 = po.srcs[0]
            o.B, o.H, o.W = pb.B, s0.H, s0.W
            o.nsrc = len(po.srcs)
            for j, s in enumerate(po.srcs):
                o.cin[j] = s.C
                if s.kind == "nchw_in":
                    self.in_slots.append((i, j))
                else:
                    o.src[j] = s.buf.data_ptr() + s.ch_off * pb._storage(s.kind)[1]
                    o.src_pitch[j] = s.pitch if s.parent is not None else 0
            if po.type == OP_HEADS:
                self._set_heads(i, o, po)
                continue
            o.cout = po.cout
            o.kh, o.kw = po.k; o.stride = po.stride; o.pad_h, o.pad_w = po.pad
            o.Hd, o.Wd, o.out_sy, o.out_sx, o.out_oy, o.out_ox = po.out_map
            o.Ho, o.Wo = po.HoWo
            o.out_ch_off = po.out_ch_off
            d = po.dst
            o.out_ch_total = d.C
            if d.kind == "nchw_out":
                self.out_slots.setdefault(d.name, []).append(i)
            else:
                o.dst = d.buf.data_ptr()
            if po.res is not None:
                o.res = po.res.buf.data_ptr()
            if po.aux is not None:
                o.aux = po.aux.buf.data_ptr()
            o.aux_pitch = po.aux_pitch
            if po.weight is not None:
                o.weight = po.weight.data_ptr()
            if po.bias is not None:
                o.bias = po.bias.data_ptr()
        if ctypes.sizeof(OpStruct) != _lib.lib().cpb200_sizeof_op():
            raise RuntimeError("cpb200_op layout mismatch between Python binding and library")
        self.n = n
        self._prepared = False
        self._done = None           # event recorded after the last run, on _last_stream (see run)
        self._last_stream = None
        self._streams = set()       # the streams the plan's memory is recorded on

    @staticmethod
    def _root(s: Sym) -> Sym:
        """the tensor that owns the storage of ``s`` (a channel slice's parent); liveness is tracked on it"""
        while s.parent is not None:
            s = s.parent
        return s

    def _readers(self, ops: Sequence[Op]) -> Dict[int, List[int]]:
        """id(root Sym) -> indices of the ops reading it, ascending"""
        readers = {}
        for i, po in enumerate(ops):
            for s in po.operands():
                readers.setdefault(id(self._root(s)), []).append(i)
        return readers

    def _prune(self, pb: PlanBuilder):
        """Split precisions emit a CONVERT back to planes after every fp32-island op; inside a chain of island ops it is
        dead.  Drop ops whose result nobody reads (outputs, externals and the program's last op are roots)."""
        if not pb.split:
            return
        ops = pb.ops
        readers = self._readers(ops)
        live = [False] * len(ops)
        for i in range(len(ops) - 1, -1, -1):
            d = self._root(ops[i].dst)
            live[i] = i == len(ops) - 1 or d.fixed or d.keep or any(live[c] for c in readers.get(id(d), ()) if c > i)
        pb.ops = [po for i, po in enumerate(ops) if live[i]]

    def _fuse_heads(self, pb: PlanBuilder):
        """Replace (tensor-core 3x3 conv + ReLU -> 1x1 conv with NCHW fp32 output) pairs over one shared input by ONE
        OP_HEADS op (csrc/net_heads.cu): the hidden maps, otherwise written by each 3x3 conv and read back once by its 1x1
        conv, stay on the chip and are never allocated.  The kernel sums the same products in the same order, so the
        outputs are bit-identical.  A pair qualifies when the 3x3 conv is stride 1 / pad 1 over one dense input of at
        most 64 channels (C % 16 == 0) and maps of at least 8 x 8, writes a multiple of 128 channels, and its result is
        read by the 1x1 conv alone; nothing involved may be marked keep."""
        if not pb.use_tc:
            return
        ops = pb.ops
        readers = self._readers(ops)
        pairs = []
        for i, a in enumerate(ops):
            if not (a.type == OP_CONV and a.flags == FLAG_TC | FLAG_RELU and a.k == (3, 3) and a.stride == 1
                    and a.pad == (1, 1) and len(a.srcs) == 1 and a.res is None and a.out_ch_off == 0):
                continue
            x, h = a.srcs[0], a.dst
            if not (x.kind == "act" and x.parent is None and x.C % 16 == 0 and x.C <= 64 and x.H >= 8 and x.W >= 8
                    and a.out_map == (x.H, x.W, 1, 1, 0, 0) and a.HoWo == (x.H, x.W)
                    and h.kind == "act" and h.parent is None and not h.keep and not h.fixed and h.C % 128 == 0):
                continue
            r = readers.get(id(h), [])
            if len(r) != 1:
                continue
            b = ops[r[0]]
            d = b.dst
            if not (b.type == OP_CONV and b.flags == FLAG_TC | FLAG_OUT_NCHW_F32 and b.k == (1, 1) and len(b.srcs) == 1
                    and b.srcs[0] is h and b.res is None and b.cout <= 48
                    and d.kind == "nchw_out" and d.C == b.cout and b.out_ch_off == 0
                    and b.out_map == (x.H, x.W, 1, 1, 0, 0) and not readers.get(id(d))):
                continue
            pairs.append((i, r[0]))
        if not pairs:
            return
        x0, hid = ops[pairs[0][0]].srcs[0], ops[pairs[0][0]].cout
        pairs = [p for p in pairs if ops[p[0]].srcs[0] is x0 and ops[p[0]].cout == hid][:8]
        first = min(i for i, _ in pairs)
        if any(self._root(po.dst) is x0 for po in ops[first:]):
            return
        heads = [(ops[i], ops[j]) for i, j in pairs]
        w = torch.stack([a.weight for a, _ in heads]).contiguous()       # [head][(plane)][tap][K-slab][hid][bk]
        bias = torch.cat([a.bias for a, _ in heads]).contiguous()
        pb.keep += [w, bias]
        fused = Op(OP_HEADS, pb.act_dtype, [x0], heads[0][1].dst, sum(b.cout for _, b in heads),
                   flags=FLAG_TC | FLAG_OUT_NCHW_F32, k=(3, 3), pad=(1, 1), weight=w, bias=bias, heads=heads)
        drop = {k for p in pairs for k in p}
        pb.ops = [fused if k == first else po for k, po in enumerate(ops) if k == first or k not in drop]

    def _set_heads(self, i: int, o: OpStruct, po: Op):
        s0 = po.srcs[0]
        o.cout = po.cout
        o.kh = o.kw = 3; o.stride = 1; o.pad_h = o.pad_w = 1
        o.Ho, o.Wo, o.Hd, o.Wd = s0.H, s0.W, s0.H, s0.W
        o.out_sy = o.out_sx = 1
        o.out_ch_total = po.cout
        tab = (HeadStruct * len(po.heads))()
        for k, (a, b) in enumerate(po.heads):
            e = tab[k]
            e.hidden, e.cout = a.cout, b.cout
            e.weight, e.bias = b.weight.data_ptr(), b.bias.data_ptr()
            e.acc_scale3, e.acc_scale1 = a.acc_scale, b.acc_scale
            self.out_slots.setdefault(b.dst.name, []).append((i, k))
        self._head_tables[i] = tab
        o.aux = ctypes.addressof(tab); o.aux_pitch = len(tab)
        o.weight = po.weight.data_ptr(); o.bias = po.bias.data_ptr()

    def _allocate(self, pb: PlanBuilder):
        """Liveness-based buffer reuse: a buffer returns to the pool after the last op that reads or writes it."""
        last_use = {}                                   # id(root sym) -> index of the last op reading or writing it
        for i, po in enumerate(pb.ops):
            for s in (*po.operands(), po.dst):
                last_use[id(self._root(s))] = i
        pool = {}
        release_at = {}
        self.buffers = []
        total = 0
        no_reuse = os.environ.get("CPB200_NO_REUSE", "0") == "1"      # diagnostics: keep every intermediate (tools/layer_err.py)
        for i, po in enumerate(pb.ops):
            d = po.dst
            if not d.fixed and d.buf is None:
                nbytes = pb.B * d.H * d.W * d.C * pb._storage(d.kind)[0]
                cand = [k for k in pool if k >= nbytes and pool[k]]
                if cand:
                    raw = pool[min(cand)].pop()
                else:
                    raw = torch.empty(nbytes, dtype=torch.uint8, device=pb.device)
                    self.buffers.append(raw); total += nbytes
                d.buf = raw
                if not d.keep:
                    release_at.setdefault(last_use[id(d)], []).append(d)
            for s in release_at.pop(i, []):
                if not no_reuse:
                    pool.setdefault(s.buf.numel(), []).append(s.buf)
        self.activation_bytes = total

    def tensor(self, sym: Sym) -> torch.Tensor:
        """An internal NHWC activation (valid until a later op reuses its buffer): a view, or — split precisions —
        the fp32 value hi + lo reassembled from the two planes."""
        pb = self.pb
        split = pb.split and sym.kind == "act"
        if sym.fixed and not split:
            return sym.buf
        slot, _, dt = pb._storage(sym.kind)
        raw = sym.buf.view(torch.uint8).view(-1) if sym.fixed else sym.buf
        t = raw[: pb.B * sym.H * sym.W * sym.C * slot].view(dt)
        if split:
            hi, lo = t.view(2, pb.B, sym.H, sym.W, sym.C)
            return hi.float() + lo.float()
        return t.view(pb.B, sym.H, sym.W, sym.C)

    def bind(self, x: torch.Tensor, outs: dict):
        """Point the program at this call's input and output tensors."""
        for (i, j) in self.in_slots:
            self.ops[i].src[j] = x.data_ptr()
        for name, idxs in self.out_slots.items():
            p = outs[name].data_ptr()
            for i in idxs:
                if isinstance(i, tuple):
                    self._head_tables[i[0]][i[1]].dst = p
                else:
                    self.ops[i].dst = p

    def run(self, stream: Optional[int] = None):
        """Enqueue the program on the current stream of the plan's device, or on ``stream`` (a raw ``cudaStream_t``
        handle of the current device) for callers that hold one.

        Every run reads and writes the plan's one set of activation buffers, so runs are ordered across streams: a run
        on another stream than the previous run's first waits for that run to end.  The first run on a stream also
        records the plan's buffers and weights on it, so when the plan is dropped the allocator does not hand their
        memory out before the work enqueued there has finished."""
        L = _lib.lib()
        if not self._prepared:
            _lib.check(L.cpb200_prepare_ops(self.ops, self.n), "cpb200_prepare_ops")
            self._prepared = True
        s = torch.cuda.current_stream(self.device) if stream is None else \
            torch.cuda.ExternalStream(stream, device=self.device)
        self._order(s)
        if stream is None:
            _lib.launch("run_ops", self.device, self.ops, self.n)
        else:
            _lib.check(L.cpb200_run_ops(self.ops, self.n, stream), "cpb200_run_ops")
        self._done.record(s)

    def _order(self, s):
        """Make stream ``s`` wait for the previous run when that ran on another stream, and record the plan's device
        memory on ``s`` the first time a run uses it."""
        if self._done is None:
            self._done = torch.cuda.Event()
        elif self._last_stream != s.cuda_stream:
            s.wait_event(self._done)
        if s.cuda_stream not in self._streams:
            self._streams.add(s.cuda_stream)
            for t in {id(t): t for t in (*self.buffers, *self.pb.keep) if t.is_cuda}.values():
                t.record_stream(s)
        self._last_stream = s.cuda_stream

    def profile_ops(self, stream: int, reps: int = 3):
        """CUDA-event time of every op launched ON ITS OWN (ms, best of ``reps``), after one full run has filled the buffers.
        Serialised launches on whatever the earlier ops left in the (recycled) buffers: per-op SHARES of a step and per-op
        rates, not a step time.  ``stream`` is the device's current stream (the events are recorded there).  Returns
        [(op type, flags, B, Ho, Wo, cout, cin_total, kh, kw, ms)]."""
        L = _lib.lib()
        self.run(stream)
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        out = []
        step = ctypes.sizeof(OpStruct)
        base = ctypes.addressof(self.ops)
        for i in range(self.n):
            one = ctypes.cast(base + i * step, ctypes.POINTER(OpStruct))
            best = None
            for _ in range(reps):
                ev0.record()
                _lib.check(L.cpb200_run_ops(one, 1, stream), "cpb200_run_ops")
                ev1.record(); ev1.synchronize()
                t = ev0.elapsed_time(ev1)
                best = t if best is None or t < best else best
            o = self.ops[i]
            out.append((int(o.type), int(o.flags), int(o.B), int(o.Ho), int(o.Wo), int(o.cout),
                        int(sum(o.cin[j] for j in range(o.nsrc))), int(o.kh), int(o.kw), best))
        return out

    def __del__(self):
        try:
            if getattr(self, "_prepared", False):
                _lib.lib().cpb200_release_ops(self.ops, self.n)
        except Exception:
            pass
