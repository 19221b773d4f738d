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
from typing import List, Optional, Sequence

import torch

from . import _lib

OP_CONV, OP_STEM, OP_MAXPOOL, OP_DWDECONV_ADD, OP_DCN, OP_IM2COL_W, OP_UPSAMPLE_ADD = 1, 2, 3, 4, 5, 6, 7
OP_DWCONV, OP_AVGPOOL, OP_SCALE_ADD, OP_CONVERT, OP_S2D = 8, 9, 10, 11, 12
FLAG_RELU, FLAG_OUT_NCHW_F32, FLAG_OUT_F32, FLAG_TC, FLAG_HSWISH, FLAG_HSIGMOID, FLAG_TO_F32 = 1, 2, 4, 8, 16, 32, 64
_ACT_FLAG = {None: 0, "relu": FLAG_RELU, "hswish": FLAG_HSWISH, "hsigmoid": FLAG_HSIGMOID}
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


class Sym:
    """Symbolic activation tensor (NHWC unless kind says otherwise)."""
    __slots__ = ("C", "H", "W", "kind", "name", "_buf", "producer", "_last_use", "fixed", "parent", "ch_off", "_f32", "_sp", "keep")

    def __init__(self, C, H, W, kind="act", name="", parent=None, ch_off=0):
        self.C, self.H, self.W, self.kind, self.name = C, H, W, kind, name
        self._buf = None         # torch tensor once allocated
        self.producer = -1
        self._last_use = -1
        self.fixed = False       # externally provided storage (network input / outputs)
        self.parent = parent     # channel slice [ch_off, ch_off + C) of `parent` (shares its storage)
        self.ch_off = ch_off
        self._f32 = None         # split precisions: cached fp32 copy / split copy of this activation
        self._sp = None
        self.keep = False        # PlanBuilder.keep_result(): never pruned, buffer never recycled (tests / diagnostics read it)

    # a slice lives in its parent's buffer and keeps the parent alive
    @property
    def buf(self):
        return self.parent.buf if self.parent is not None else self._buf

    @buf.setter
    def buf(self, v):
        self._buf = v

    @property
    def last_use(self):
        return self.parent.last_use if self.parent is not None else self._last_use

    @last_use.setter
    def last_use(self, v):
        if self.parent is not None:
            self.parent.last_use = v
        else:
            self._last_use = v

    @property
    def pitch(self):
        return self.parent.C if self.parent is not None else self.C


class _PendingOp:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def fold_bn(w: torch.Tensor, b: Optional[torch.Tensor], bn: Optional[dict]):
    """conv weight (Co,Ci,kh,kw) [+bias] followed by eval BatchNorm -> equivalent weight/bias."""
    w = w.float()
    co = w.shape[0]
    b = torch.zeros(co, device=w.device) if b is None else b.float()
    if bn is None:
        return w, b
    scale = bn["weight"].float() / torch.sqrt(bn["running_var"].float() + BN_EPS)
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
        self.ops: List[_PendingOp] = []
        self.keep: List[torch.Tensor] = []      # weights / biases kept alive
        self.syms: List[Sym] = []
        # tensor-core (wgmma) path: 16-bit operands only; CPB200_TC=0 forces the SIMT kernels (bf16: debugging)
        if tc is None:
            tc = os.environ.get("CPB200_TC", "1") != "0"
        if self.split and not tc:
            raise ValueError("split precisions run on the tensor-core path only")
        self.use_tc = bool(tc) and precision != "fp32"

    # ---- symbolic tensors -------------------------------------------------------------
    def _sym(self, C, H, W, kind="act", name=""):
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
        self._root_of(s).keep = True
        return s

    @staticmethod
    def _root_of(s: Sym) -> Sym:
        while s.parent is not None:
            s = s.parent
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
            pf = self._to_f32(x.parent)
            v = Sym(x.C, x.H, x.W, "actf32", parent=pf, ch_off=x.ch_off)
            v.producer = pf.producer
            return v
        if x._f32 is None:
            y = self._sym(x.C, x.H, x.W, "actf32", x.name + ".f32")
            self._emit(_PendingOp(type=OP_CONVERT, flags=FLAG_TO_F32, k=(1, 1), stride=1, pad=(0, 0), weight=None, bias=None,
                                  cout=x.C, dtype=self.act_dtype), [x], y)
            x._f32 = y; y._sp = x
        return x._f32

    def _to_split(self, y: Sym) -> Sym:
        """split copy of an fp32 NHWC activation produced inside an fp32 island."""
        if not self.split or y.kind != "actf32":
            return y
        if y._sp is None:
            x = self._sym(y.C, y.H, y.W, "act", y.name + ".sp")
            self._emit(_PendingOp(type=OP_CONVERT, flags=0, k=(1, 1), stride=1, pad=(0, 0), weight=None, bias=None,
                                  cout=y.C, dtype=self.act_dtype), [y], x)
            y._sp = x; x._f32 = y
        return y._sp

    def _island_sym(self, C, H, W):
        """output of an op that runs on fp32 in split mode (kind 'actf32'), an ordinary activation otherwise."""
        return self._sym(C, H, W, "actf32" if self.split else "act")

    def _emit(self, op: _PendingOp, srcs: Sequence[Sym], dst: Sym, extra: Sequence[Optional[Sym]] = ()):
        if not hasattr(op, "dtype"):
            op.dtype = self.act_dtype
        if not hasattr(op, "acc_scale"):
            op.acc_scale = 1.0
        idx = len(self.ops)
        for s in list(srcs) + [e for e in extra if e is not None]:
            s.last_use = max(s.last_use, idx)
        if dst.producer < 0:
            dst.producer = idx
        dst.last_use = max(dst.last_use, idx)
        op.srcs, op.dst, op.extra = list(srcs), dst, list(extra)
        self.ops.append(op)

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

    def _pack_conv_tc(self, w: torch.Tensor, bk: int):
        """(Co,Ci,kh,kw) fp32 -> wgmma layout [kh*kw][Ci/bk][Co_pad16][bk] bf16 (K-major B operand, slab-major:
        the rows of one (tap, K-slab) block are contiguous, so a TMA weight box is one dense run of memory instead of
        Co rows strided by Ci).  bk = the kernels' K-slab width."""
        co, ci, kh, kw = w.shape
        assert ci % bk == 0
        cop = (co + 15) // 16 * 16
        p = torch.zeros(kh * kw, ci // bk, cop, bk, dtype=torch.float32, device=w.device)
        p[:, :, :co, :] = w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci // bk, bk).permute(0, 2, 1, 3)
        if self.split:
            # [plane][tap][slab][Co_pad][bk]: hi plane then lo plane; fp16 planes carry the weights times a power of two
            # (pow2_scale) whose inverse the kernel applies to the accumulator (cpb200_op.acc_scale)
            self._last_scale = pow2_scale(w) if self.torch16 == torch.float16 else 1.0
            t = split_planes(p * self._last_scale, self.torch16).to(self.device)
            self.keep.append(t)
            return t
        self._last_scale = 1.0
        return self._dev(p, torch.bfloat16)

    @staticmethod
    def _tc_bk(srcs) -> int:
        """K-slab width the tensor-core kernels use for these inputs (csrc/net_tc.cu, net_tc3.cu: 64 / 32 / 16)."""
        bk = 64
        for s in srcs:
            if s.C % 64:
                bk = min(bk, 32 if s.C % 32 == 0 else 16)
        return bk

    def channel_slice(self, x: Sym, off: int, c: int) -> Sym:
        """View of channels [off, off+c) of an NHWC activation (no copy): readable by conv ops through the op's
        ``src_pitch`` field.  Used to feed the six head 1x1 convs from ONE fused hidden tensor."""
        assert x.parent is None and x.kind == "act" and 0 <= off and off + c <= x.C and off % 16 == 0 and c % 16 == 0
        v = Sym(c, x.H, x.W, "act", parent=x, ch_off=off)
        v.producer = x.producer
        return v

    def _pack_stem_tc(self, w: torch.Tensor):
        """(N,3,7,7) fp32 -> the 128-byte-swizzled K-major B operand image of csrc/net_stem_tc.cu:
        k = (c*7 + r)*8 + s (s = 7 and k >= 168 are zero), three 64-wide slabs of N rows x 128 bytes,
        16-byte chunk j of row n stored at chunk j ^ (n & 7)."""
        N = w.shape[0]
        wk = torch.zeros(N, 3, 7, 8, dtype=torch.float32, device=w.device)
        wk[..., :7] = w.float()
        wk = torch.nn.functional.pad(wk.reshape(N, 168), (0, 24))                   # (N, 192)
        blk = wk.reshape(N, 3, 8, 8).permute(1, 0, 2, 3)                            # [slab][n][chunk j][e]
        n_idx = torch.arange(N, device=w.device).view(1, N, 1, 1).expand(3, N, 8, 8)
        j_idx = torch.arange(8, device=w.device).view(1, 1, 8, 1).expand(3, N, 8, 8)
        img = torch.zeros(3, N, 8, 8, dtype=torch.float32, device=w.device)
        img.scatter_(2, (j_idx ^ (n_idx & 7)), blk.contiguous())
        return self._dev(img, torch.bfloat16)

    def _pack_stem_tc_h(self, w: torch.Tensor):
        """(N,3,7,7) fp32 -> B operand image of the stride-1 tensor-core stem (stem_tc_h_kernel): one block per
        horizontal tap s of N rows x 64 bytes, k = c*7 + r (21 real of 32), 64-byte swizzle: 16-byte chunk j of
        row n stored at chunk j ^ ((n >> 1) & 3) (tap blocks are multiples of 1024 bytes)."""
        N = w.shape[0]
        wk = torch.zeros(7, N, 32, dtype=torch.float32, device=w.device)                # [s][n][k]
        wk[:, :, :21] = w.float().permute(3, 0, 1, 2).reshape(7, N, 21)
        blk = wk.reshape(7, N, 4, 8)                                                     # [s][n][chunk j][e]
        n_idx = torch.arange(N, device=w.device).view(1, N, 1, 1).expand(7, N, 4, 8)
        j_idx = torch.arange(4, device=w.device).view(1, 1, 4, 1).expand(7, N, 4, 8)
        img = torch.zeros(7, N, 4, 8, dtype=torch.float32, device=w.device)
        if self.split:
            # per tap [hi tile (N rows) | lo tile (N rows)]; row n' = plane * N + n of the 2N-row block is swizzled with
            # (n' >> 1) & 3 == (n >> 1) & 3 (N is a multiple of 8)
            self._last_scale = pow2_scale(w) if self.torch16 == torch.float16 else 1.0
            planes = split_planes(blk * self._last_scale, self.torch16).float()       # (2, 7, N, 4, 8)
            out = torch.zeros(7, 2, N, 4, 8, dtype=torch.float32, device=w.device)
            for pl in range(2):
                tmp = torch.zeros(7, N, 4, 8, dtype=torch.float32, device=w.device)
                tmp.scatter_(2, (j_idx ^ ((n_idx >> 1) & 3)), planes[pl].contiguous())
                out[:, pl] = tmp
            t = out.to(self.torch16).to(self.device).contiguous()
            self.keep.append(t)
            return t
        self._last_scale = 1.0
        img.scatter_(2, (j_idx ^ ((n_idx >> 1) & 3)), blk.contiguous())
        return self._dev(img, torch.bfloat16)

    def _tc_ok(self, srcs, co, kh, kw, stride, out, out_map, Wo):
        return (self.use_tc and stride in (1, 2) and Wo >= 8
                and all(s.C % 16 == 0 and s.kind == "act" for s in srcs)
                and (co % 16 == 0 or out in ("f32", "nchw")) and kh * kw <= 49)

    # ---- ops -------------------------------------------------------------------------------
    # Split precisions (bf16x2 / fp16x2): convs, DCNs and the stride-1 stem run natively on the hi/lo planes (tensor-core
    # kernels), max-pool and the IDAUp depthwise upsample have split kernels; everything else (and conv shapes the
    # tensor-core kernels do not take, e.g. maps narrower than 8 pixels) runs on fp32 between two CONVERT ops — an
    # "fp32 island": slower, never less precise.
    def stem(self, x: Sym, w, b, k, stride, pad, relu=True, act=None):
        co, ci = w.shape[0], w.shape[1]
        mode = os.environ.get("CPB200_TC_STEM", "1")
        if (self.use_tc and not self.split and mode == "im2col" and stride == 1 and k * ci <= 32 and co % 16 == 0 and pad == k // 2):
            # first tensor-core stem (kept for the record, CPB200_TC_STEM=im2col): gather the k horizontal taps of
            # every pixel into 32 channels IN HBM, then a k x 1 conv with K = k * 32 on the halo-reuse kernel.
            # Correct (tests/test_net_gpu.py::test_stem_im2col_path) but measured SLOWER than the CUDA-core stem at
            # B=32 512x512 (1430 us vs 1045 us: 537 MB intermediate + 65 536 N=16 tiles).
            t = self._sym(32, x.H, x.W)
            self._emit(_PendingOp(type=OP_IM2COL_W, flags=0, k=(1, k), stride=1, pad=(0, pad), weight=None,
                                  bias=None, cout=32), [x], t)
            w2 = torch.zeros(co, 32, k, 1, dtype=torch.float32, device=w.device)
            # w2[o, s*ci + c, r, 0] = w[o, c, r, s]
            w2[:, :k * ci, :, 0] = w.float().permute(0, 3, 1, 2).reshape(co, k * ci, k)
            return self.conv([t], w2, b.float(), stride=1, relu=relu, pad_hw=(pad, 0))
        if (self.use_tc and self.split and mode != "0" and stride == 2 and ci == 3 and k in (3, 7) and pad == k // 2
                and co % 16 == 0 and x.H % 2 == 0 and x.W % 2 == 0 and x.kind == "nchw_in"
                and os.environ.get("CPB200_S2D_STEM", "1") != "0"):
            # Stride-2 stems in split precisions (ResNet 7x7, HRNet 3x3): space-to-depth of the image (OP_S2D: 2x2 pixel
            # blocks -> 12 of 16 channels) turns  out[o] = sum_r w[r] x[2o - pad + r]  into a STRIDE-1 conv over the half-
            # resolution map: input index 2o - pad + r = 2 (o + q) + parity with q = floor((r - pad) / 2), parity =
            # (r - pad) & 1, so a 7-tap filter becomes taps q = -2..1 (a 5x5 conv, pad 2, last tap zero) and a 3-tap filter
            # q = -1..0 (a 3x3 conv, pad 1).  It then runs on the split tensor-core halo kernel instead of a CUDA-core
            # fp32 island (ResNet-50 B=16: 954 us + a CONVERT pass).
            z = self._sym(16, x.H // 2, x.W // 2)
            self._emit(_PendingOp(type=OP_S2D, flags=0, k=(2, 2), stride=2, pad=(0, 0), weight=None, bias=None, cout=16), [x], z)
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
        if (self.use_tc and mode != "0" and k == 7 and ci == 3 and pad == 3 and stride in (1, 2) and co in (16, 64)
                and not (self.split and stride != 1)):
            # tensor-core stem with the im2col done in shared memory (csrc/net_stem_tc.cu); split precisions: stride 1 only
            y = self._sym(co, Ho, Wo)
            wp = self._pack_stem_tc_h(w) if stride == 1 else self._pack_stem_tc(w)
            self._emit(_PendingOp(type=OP_STEM, flags=flags | FLAG_TC, k=(k, k), stride=stride, pad=(pad, pad),
                                  weight=wp, bias=self._dev(b), cout=co,
                                  acc_scale=(rz_compensation(self.precision, 7 * 32) / getattr(self, "_last_scale", 1.0))
                                  if (stride == 1 and self.split) else 1.0), [x], y)
            return y
        y = self._island_sym(co, Ho, Wo)
        wp = self._dev(w.permute(2, 3, 1, 0).reshape(k * k * ci, co))
        self._emit(_PendingOp(type=OP_STEM, flags=flags, k=(k, k), stride=stride,
                              pad=(pad, pad), weight=wp, bias=self._dev(b), cout=co,
                              dtype=F32 if self.split else self.act_dtype), [x], y)
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
        flags = _ACT_FLAG[act] if act else (FLAG_RELU if relu else 0)     # act: 'relu' | 'hswish' | 'hsigmoid'
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
        wp = self._pack_conv_tc(w, self._tc_bk(srcs)) if tc else self._pack_conv(w)
        self._emit(_PendingOp(type=OP_CONV, flags=flags, k=(kh, kw), stride=stride, pad=(ph, pw),
                              weight=wp, bias=self._dev(b), cout=co, ch_off=ch_off,
                              out_map=(Hd, Wd, sy, sx, oy, ox), HoWo=(Ho, Wo), w_raw=w,
                              dtype=F32 if island else self.act_dtype,
                              acc_scale=(rz_compensation(self.precision, kh * kw * ci) / self._last_scale) if (tc and self.split) else 1.0),
                   srcs, y, [res])
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

    def maxpool(self, x: Sym, k=2, stride=2, pad=0):
        Ho = (x.H + 2 * pad - k) // stride + 1; Wo = (x.W + 2 * pad - k) // stride + 1
        y = self._sym(x.C, Ho, Wo)
        self._emit(_PendingOp(type=OP_MAXPOOL, flags=0, k=(k, k), stride=stride, pad=(pad, pad),
                              weight=None, bias=None, cout=x.C), [x], y)
        return y

    def up_add(self, x: Sym, skip: Optional[Sym], w):
        """depthwise ConvTranspose2d weight (C,1,2f,2f), stride f, pad f//2, + skip."""
        C, _, k, _ = w.shape
        f = k // 2
        Ho = (x.H - 1) * f - 2 * (f // 2) + k; Wo = (x.W - 1) * f - 2 * (f // 2) + k
        y = self._sym(C, Ho, Wo)
        wp = self._dev(w.float().reshape(C, k * k).t())          # [k*k][C]
        self._emit(_PendingOp(type=OP_DWDECONV_ADD, flags=0, k=(k, k), stride=f, pad=(f // 2, f // 2),
                              weight=wp, bias=None, cout=C), [x], y, [skip])
        return y

    def _f32_op(self, op: _PendingOp, srcs, C, H, W, extra=()):
        """emit an op that has no split kernel: on fp32 between CONVERT ops in split mode, natively otherwise."""
        if self.split:
            op.dtype = F32
            srcs = [self._to_f32(s_) for s_ in srcs]
            extra = [self._to_f32(e) for e in extra]
        y = self._island_sym(C, H, W)
        self._emit(op, srcs, y, list(extra))
        return self._to_split(y)

    def _native_split(self, *syms) -> bool:
        """split mode and every operand a whole split-plane tensor: the element-wise kernels then read / write the planes
        directly (csrc/net_simt.cu: SpC / SpM handles) and no fp32 island is needed."""
        return self.split and all(s is None or (s.kind == "act" and s.parent is None) for s in syms)

    def dwconv(self, x: Sym, w, b, stride=1, act=None):
        """depthwise conv, w (C,1,k,k) BN-folded, pad k//2   (mobilenetv3.py:124-127)."""
        C, _, k, _ = w.shape
        assert C == x.C
        Ho = (x.H + 2 * (k // 2) - k) // stride + 1; Wo = (x.W + 2 * (k // 2) - k) // stride + 1
        wp = self._dev(w.float().reshape(C, k * k).t())          # [k*k][C]
        op = _PendingOp(type=OP_DWCONV, flags=_ACT_FLAG[act], k=(k, k), stride=stride, pad=(k // 2, k // 2),
                        weight=wp, bias=self._dev(b), cout=C)
        if self._native_split(x):
            y = self._sym(C, Ho, Wo, "act")
            self._emit(op, [x], y)
            return y
        return self._f32_op(op, [x], C, Ho, Wo)

    def avgpool(self, x: Sym):
        """global average pool -> (C, 1, 1)   (mobilenetv3.py:100).  Split mode: planes in, fp32 out (the 1x1-map SE convs
        that follow run on fp32 anyway)."""
        op = _PendingOp(type=OP_AVGPOOL, flags=0, k=(x.H, x.W), stride=1, pad=(0, 0), weight=None, bias=None, cout=x.C)
        if self._native_split(x):
            y = self._island_sym(x.C, 1, 1)
            self._emit(op, [x], y)
            return self._to_split(y)                                # dead unless someone wants the planes; pruned
        return self._f32_op(op, [x], x.C, 1, 1)

    def scale_add(self, x: Sym, gate: Sym, skip: Optional[Sym] = None):
        """x * gate[b, c] (+ skip)   (mobilenetv3.py:111,146).  Split mode: x / skip / result are planes, the gate is fp32."""
        assert gate.C == x.C and gate.H == 1 and gate.W == 1
        op = _PendingOp(type=OP_SCALE_ADD, flags=0, k=(1, 1), stride=1, pad=(0, 0), weight=None, bias=None, cout=x.C)
        if self._native_split(x, skip) and gate.parent is None:
            y = self._sym(x.C, x.H, x.W, "act")
            self._emit(op, [x], y, [self._to_f32(gate), skip])
            return y
        return self._f32_op(op, [x], x.C, x.H, x.W, [gate, skip])

    def upsample_add(self, x: Sym, skip: Optional[Sym], f: int, relu=False):
        """nearest-neighbour upsample x f of ``x`` (+ skip)(+ReLU)   (pose_higher_hrnet.py:186-187,224-232)."""
        op = _PendingOp(type=OP_UPSAMPLE_ADD, flags=FLAG_RELU if relu else 0, k=(1, 1), stride=f, pad=(0, 0),
                        weight=None, bias=None, cout=x.C)
        if self._native_split(x, skip):
            y = self._sym(x.C, x.H * f, x.W * f, "act")
            self._emit(op, [x], y, [skip])
            return y
        return self._f32_op(op, [x], x.C, x.H * f, x.W * f, [skip])

    def dcn(self, x: Sym, w, b, om_w, om_b, relu=True):
        """DCN module (dcn_v2.py:117-127) with BN already folded into (w, b)."""
        # offset/mask conv: 27 channels padded to 32 so every pixel row is 128 bytes (vector stores / loads)
        om_w32 = torch.zeros(32, *om_w.shape[1:], dtype=torch.float32, device=om_w.device); om_w32[:27] = om_w.float()
        om_b32 = torch.zeros(32, dtype=torch.float32, device=om_b.device); om_b32[:27] = om_b.float()
        om = self.conv([x], om_w32, om_b32, stride=1, pad=1, relu=False, out="f32")
        co = w.shape[0]
        tc = (self.use_tc and x.kind == "act" and x.C % 64 == 0 and co % 16 == 0 and 32 <= co and x.W >= 8
              and os.environ.get("CPB200_TC_DCN", "1") != "0")
        island = self.split and not tc
        xin = self._to_f32(x) if island else x
        y = self._sym(co, x.H, x.W, "actf32" if island else "act")
        wp = self._pack_conv_tc(w, 64) if tc else self._pack_conv(w)
        self._emit(_PendingOp(type=OP_DCN, flags=(FLAG_RELU if relu else 0) | (FLAG_TC if tc else 0), k=(3, 3),
                              stride=1, pad=(1, 1), weight=wp, bias=self._dev(b), cout=co, w_raw=w,
                              dtype=F32 if island else self.act_dtype,
                              acc_scale=(rz_compensation(self.precision, 9 * x.C) / self._last_scale) if (tc and self.split) else 1.0),
                   [xin], y, [om])
        return self._to_split(y) if island else y

    # ---- finalisation -----------------------------------------------------------------------
    def build(self) -> "Plan":
        return Plan(self)


def _esize(pb: "PlanBuilder", kind: str) -> int:
    """bytes per ELEMENT SLOT of an NHWC tensor of this kind (split activations: two 16-bit planes)."""
    if kind in ("f32", "actf32"):
        return 4
    if kind == "act":
        return 4 if (pb.act_dtype == F32 or pb.split) else 2
    raise KeyError(kind)


def _ptr_esize(pb: "PlanBuilder", kind: str) -> int:
    """bytes per element for pointer arithmetic inside ONE plane (channel-slice offsets)."""
    if kind in ("f32", "actf32"):
        return 4
    return 4 if pb.act_dtype == F32 else 2


class Plan:
    """Allocated, ready-to-run op program for one (B, H, W, precision)."""

    def __init__(self, pb: PlanBuilder):
        self.pb = pb
        self.device = pb.device
        self._prune(pb)
        self._allocate(pb)
        n = len(pb.ops)
        self.ops = (OpStruct * n)()
        self.in_slots = []      # (op index, src slot) fed by the network input
        self.out_slots = {}     # output name -> list of op indices writing it
        for i, po in enumerate(pb.ops):
            o = self.ops[i]
            o.type = po.type; o.flags = po.flags; o.act_dtype = po.dtype
            o.acc_scale = float(getattr(po, "acc_scale", 1.0))
            s0 = po.srcs[0]
            o.B, o.H, o.W = pb.B, s0.H, s0.W
            o.nsrc = len(po.srcs)
            for j, s in enumerate(po.srcs):
                o.cin[j] = s.C
                if s.kind == "nchw_in":
                    self.in_slots.append((i, j))
                else:
                    o.src[j] = s.buf.data_ptr() + s.ch_off * _ptr_esize(pb, s.kind)
                    o.src_pitch[j] = s.pitch if s.parent is not None else 0
            o.cout = po.cout
            o.kh, o.kw = po.k; o.stride = po.stride; o.pad_h, o.pad_w = po.pad
            d = po.dst
            if po.type == OP_CONV:
                o.Hd, o.Wd, o.out_sy, o.out_sx, o.out_oy, o.out_ox = po.out_map
                o.Ho, o.Wo = po.HoWo
            else:
                o.Ho, o.Wo, o.Hd, o.Wd = d.H, d.W, d.H, d.W
                o.out_sy = o.out_sx = 1
            o.out_ch_off = getattr(po, "ch_off", 0)
            o.out_ch_total = d.C
            if d.kind == "nchw_out":
                self.out_slots.setdefault(d.name, []).append(i)
            else:
                o.dst = d.buf.data_ptr()
            ex = po.extra
            if po.type == OP_CONV and ex and ex[0] is not None:
                o.res = ex[0].buf.data_ptr()
            if po.type in (OP_DCN, OP_DWDECONV_ADD, OP_UPSAMPLE_ADD) and ex and ex[0] is not None:
                o.aux = ex[0].buf.data_ptr()
                o.aux_pitch = ex[0].C
            if po.type == OP_SCALE_ADD:
                o.res = ex[0].buf.data_ptr()
                if ex[1] is not None:
                    o.aux = ex[1].buf.data_ptr()
            if po.weight is not None:
                o.weight = po.weight.data_ptr()
            if po.bias is not None:
                o.bias = po.bias.data_ptr()
        if ctypes.sizeof(OpStruct) != _lib.lib().cpb200_sizeof_op():
            raise RuntimeError("cpb200_op layout mismatch between Python binding and library")
        self.n = n
        self._prepared = False

    @staticmethod
    def _root(s: Sym) -> Sym:
        while s.parent is not None:
            s = s.parent
        return s

    def _prune(self, pb: PlanBuilder):
        """Split precisions emit a CONVERT back to planes after every fp32-island op; inside a chain of island ops it is
        dead.  Drop ops whose result nobody reads (outputs, externals and the program's last op are roots) and recompute
        the producer / last-use indices the allocator works from."""
        if not pb.split:
            return
        ops = pb.ops
        consumers = {}                                  # id(root sym) -> op indices reading it
        for i, po in enumerate(ops):
            for s in list(po.srcs) + [e for e in po.extra if e is not None]:
                consumers.setdefault(id(self._root(s)), []).append(i)
        live = [False] * len(ops)
        for i in range(len(ops) - 1, -1, -1):
            d = self._root(ops[i].dst)
            live[i] = i == len(ops) - 1 or d.fixed or d.keep or any(live[c] for c in consumers.get(id(d), ()) if c > i)
        pb.ops = [po for i, po in enumerate(ops) if live[i]]
        for s in pb.syms:
            s.producer = -1
            if s.parent is None:
                s._last_use = -1
        for i, po in enumerate(pb.ops):
            for s in list(po.srcs) + [e for e in po.extra if e is not None]:
                s.last_use = max(s.last_use, i)
            d = po.dst
            if d.producer < 0:
                d.producer = i
            d.last_use = max(d.last_use, i)

    def _allocate(self, pb: PlanBuilder):
        """Liveness-based buffer reuse: a buffer returns to the pool after its last consumer."""
        pool = {}
        release_at = {}
        self.buffers = []
        total = 0
        no_reuse = os.environ.get("CPB200_NO_REUSE", "0") == "1"      # diagnostics: keep every intermediate (tools/layer_err.py)
        for i, po in enumerate(pb.ops):
            d = po.dst
            if not d.fixed and d.buf is None:
                nbytes = pb.B * d.H * d.W * d.C * _esize(pb, d.kind)
                cand = [k for k in pool if k >= nbytes and pool[k]]
                if cand:
                    raw = pool[min(cand)].pop()
                else:
                    raw = torch.empty(nbytes, dtype=torch.uint8, device=pb.device)
                    self.buffers.append(raw); total += nbytes
                d.buf = raw
                if not d.keep:
                    release_at.setdefault(d.last_use, []).append(d)
            for s in release_at.pop(i, []):
                if not no_reuse:
                    pool.setdefault(s.buf.numel(), []).append(s.buf)
        self.activation_bytes = total

    def tensor(self, sym: Sym) -> torch.Tensor:
        """An internal NHWC activation (valid until a later op reuses its buffer): a view, or — split precisions —
        the fp32 value hi + lo reassembled from the two planes."""
        pb = self.pb
        n = pb.B * sym.H * sym.W * sym.C
        if pb.split and sym.kind == "act":
            raw = sym.buf if not sym.fixed else sym.buf.view(torch.uint8).view(-1)
            planes = raw[: 4 * n].view(pb.torch16).view(2, pb.B, sym.H, sym.W, sym.C)
            return planes[0].float() + planes[1].float()
        if sym.fixed:
            return sym.buf
        dt = torch.float32 if (sym.kind in ("f32", "actf32") or pb.act_dtype == F32) else torch.bfloat16
        return sym.buf[: n * (4 if dt == torch.float32 else 2)].view(dt).view(pb.B, sym.H, sym.W, sym.C)

    def bind(self, x: torch.Tensor, outs: dict):
        """Point the program at this call's input and output tensors."""
        for (i, j) in self.in_slots:
            self.ops[i].src[j] = x.data_ptr()
        for name, idxs in self.out_slots.items():
            p = outs[name].data_ptr()
            for i in idxs:
                self.ops[i].dst = p

    def run(self, stream: int):
        L = _lib.lib()
        if not self._prepared:
            _lib.check(L.cpb200_prepare_ops(self.ops, self.n), "prepare_ops")
            self._prepared = True
        _lib.check(L.cpb200_run_ops(self.ops, ctypes.c_int(self.n), ctypes.c_void_p(stream)), "run_ops")

    def profile_ops(self, stream: int, reps: int = 3):
        """CUDA-event time of every op launched ON ITS OWN (ms, best of ``reps``), after one full run has filled the buffers.
        Serialised launches on whatever the earlier ops left in the (recycled) buffers: per-op SHARES of a step and per-op
        rates, not a step time.  Returns [(op type, flags, B, Ho, Wo, cout, cin_total, kh, kw, ms)]."""
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
                _lib.check(L.cpb200_run_ops(one, ctypes.c_int(1), ctypes.c_void_p(stream)), "run_ops")
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
