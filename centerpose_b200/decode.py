"""Host-side mirror of the reference's decode module (``lib/models/decode.py``).

``multi_pose_decode`` keeps the reference signature and semantics
(``lib/models/decode.py:235-308``) but is ONE fused CUDA kernel launched through the C ABI
(``cpb200_multi_pose_decode``, ``include/centerpose_b200.h``).  CUDA tensors only — there
is no CPU path in the product.
"""
from __future__ import annotations

import torch

from . import _lib

_ws_cache = {}


def _workspace(device, B, J, K):
    """The zero-filled decode workspace of (device, current stream, B, J, K) and its cache key."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream, B, J, K)
    ws = _ws_cache.get(key)
    if ws is None:
        nbytes = _lib.lib().cpb200_decode_workspace_bytes(B, J, K)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)   # zero ONCE; kernel self-cleans
        if len(_ws_cache) > 64:
            _ws_cache.clear()
        _ws_cache[key] = ws
    return key, ws


def _prep(t, name, shape=None):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"multi_pose_decode: `{name}` must be a CUDA tensor "
                           "(centerpose_b200 has no CPU decode path)")
    if t.dtype != torch.float32:
        t = t.float()
    if not t.is_contiguous():
        t = t.contiguous()
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise RuntimeError(f"multi_pose_decode: `{name}` has shape {tuple(t.shape)}, expected {tuple(shape)}")
    return t


def multi_pose_decode(heat, wh, kps, reg=None, hm_hp=None, hp_offset=None, K=100,
                      apply_sigmoid=False, out=None, affine=None):
    """Same contract as the reference (``decode.py:235-236``): ``heat``/``hm_hp`` already
    sigmoid'ed (unless ``apply_sigmoid=True`` — additive: the kernel then applies the logistic
    itself, replacing ``multi_pose.py:35-37``), returns ``(B, K, 5+3J)`` fp32 on the input device.
    ``affine`` (additive): ``(B, 6)`` fp32 device tensor of per-image 2x3 matrices; when given, box corners
    and keypoints come out in original-image pixels (``post_process`` fused, see :func:`affine_for_meta`).
    """
    heat = _prep(heat, "heat")
    if heat.dim() != 4:
        raise RuntimeError("multi_pose_decode: heat must be (B,C,H,W)")
    B, cat, H, W = heat.shape
    if cat != 1:
        raise RuntimeError("multi_pose_decode: only NUM_CLASSES == 1 is supported (person), got %d" % cat)
    kps = _prep(kps, "kps")
    J = kps.shape[1] // 2
    kps = _prep(kps, "kps", (B, 2 * J, H, W))
    wh = _prep(wh, "wh", (B, 2, H, W))
    reg = _prep(reg, "reg", (B, 2, H, W))
    if hm_hp is None:
        # the reference raises here too: decode.py:307 uses hm_score unconditionally
        raise NameError("name 'hm_score' is not defined")
    hm_hp = _prep(hm_hp, "hm_hp", (B, J, H, W))
    hp_offset = _prep(hp_offset, "hp_offset", (B, 2, H, W))
    K = int(K)
    if K > H * W:
        raise RuntimeError("selected index k out of range")   # torch.topk's message
    dev = heat.device
    if out is None:
        out = torch.empty((B, K, 5 + 3 * J), dtype=torch.float32, device=dev)
    key, ws = _workspace(dev, B, J, K)
    if affine is None:
        name, extra = "multi_pose_decode", ()
    else:
        name, extra = "multi_pose_decode_affine", (_prep(affine, "affine", (B, 6)),)
    try:
        _lib.launch(name, dev, heat, wh, kps, reg, hm_hp, hp_offset, *extra, out, B, H, W, J, K,
                    1 if apply_sigmoid else 0, ws, ws.numel())
    except RuntimeError:
        # a failed / aborted launch may leave the workspace's pair counters non-zero: never reuse it
        _ws_cache.pop(key, None)
        raise
    return out


def affine_for_meta(metas, scale=1.0):
    """Host helper: per-image 2x3 matrices (float32 (B,6)) that map output-grid coordinates to original-image
    pixels — ``get_affine_transform(c, s, 0, (out_w, out_h), inv=1)`` (``lib/utils/image.py:27-60``) divided by
    the test ``scale`` (``multi_pose.py:68-69``)."""
    import numpy as np
    from .image import get_affine_transform
    rows = []
    for m in metas:
        t = get_affine_transform(m["c"], m["s"], 0, (m["out_width"], m["out_height"]), inv=1) / float(scale)
        rows.append(np.asarray(t, np.float64).reshape(6))
    return torch.from_numpy(np.stack(rows).astype(np.float32))


def sigmoid_(x: torch.Tensor) -> torch.Tensor:
    """In-place logistic on a CUDA fp32 tensor (``multi_pose.py:35-37`` ``hm.sigmoid_()``)."""
    if not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous():
        raise RuntimeError("sigmoid_: contiguous CUDA fp32 tensor required")
    _lib.launch("sigmoid_inplace", x.device, x, x.numel())
    return x


def flip_perm(flip_idx, J=17):
    """[[1,2],[3,4],...] -> the joint permutation that swaps every listed pair."""
    perm = list(range(J))
    for a, b in flip_idx:
        perm[a], perm[b] = perm[b], perm[a]
    return perm


def flip_merge(hm, wh, hps, hm_hp, flip_idx):
    """Flip-test averaging (``multi_pose.py:45-53`` with ``flip_tensor`` / ``flip_lr`` / ``flip_lr_off``,
    ``lib/models/utils.py:27-47``) in one CUDA pass.  Inputs are the fp32 NCHW head maps of ``2P`` images ordered
    ``[image, mirrored image]`` per pair (sigmoid already applied where the reference applies it); returns
    ``(hm, wh, hps, hm_hp)`` of ``P`` images.  ``hm_hp`` may be ``None``."""
    import ctypes
    tens = [hm, wh, hps] + ([hm_hp] if hm_hp is not None else [])
    for t in tens:
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4):
            raise RuntimeError("flip_merge: contiguous CUDA fp32 NCHW tensors required")
    B2, CH, H, W = hm.shape
    if B2 % 2:
        raise RuntimeError("flip_merge: batch must hold [image, mirrored image] pairs")
    P, J = B2 // 2, hps.shape[1] // 2
    if wh.shape != (B2, 2, H, W) or hps.shape != (B2, 2 * J, H, W) or (hm_hp is not None and hm_hp.shape != (B2, J, H, W)):
        raise RuntimeError("flip_merge: inconsistent head-map shapes")
    outs = [torch.empty((P,) + tuple(t.shape[1:]), dtype=torch.float32, device=hm.device) for t in tens]
    perm = (ctypes.c_int * J)(*flip_perm(flip_idx, J))
    _lib.launch("flip_merge", hm.device, hm, wh, hps, hm_hp, outs[0], outs[1], outs[2],
                outs[3] if hm_hp is not None else None, P, H, W, J, CH, perm)
    return outs[0], outs[1], outs[2], (outs[3] if hm_hp is not None else None)
