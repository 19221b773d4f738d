"""Host side of the heat-map views: what ``MultiPoseDetector.debug`` shows with ``DEBUG >= 2`` (the reference's
``Debugger.gen_colormap`` / ``gen_colormap_hp`` blended onto the network input by ``add_blend_img``) turned into the
table of ``cpb200_heatmap_views_batch`` (``csrc/heatmaps.cu``), which makes both views on the device byte for byte as
the reference's numpy and cv2 code does.

Per image the table holds the device addresses of its normalized (3, H, W) input, its (1, h, w) centre heat map and
its (C, h, w) keypoint heat maps, their sizes and where its views and its workspace go.  The inputs are checked here,
before any launch, since the kernels trust the table.
"""
from __future__ import annotations

import numpy as np
import torch

from .render import JOINT_COLORS, theme_color

VIEWS = ("pred_hm", "pred_hmhp")
MAX_C = len(JOINT_COLORS)

IMAGE = np.dtype([("input", "<u8"), ("hm", "<u8"), ("hm_hp", "<u8"), ("out_offset", "<i8"), ("ws_offset", "<i8"),
                  ("H", "<i4"), ("W", "<i4"), ("h", "<i4"), ("w", "<i4"), ("C", "<i4"), ("dr", "<i4")])
assert IMAGE.itemsize == 64


def colors(theme):
    """The (1 + 17, 3) float32 colours of the hm map and of each joint's map, as ``gen_colormap`` / ``gen_colormap_hp``
    use them: the 'white' theme inverts them (``theme_color`` already holds the inverted hm colour)."""
    hp = np.array(JOINT_COLORS, np.float32)
    if theme == "white":
        hp = np.float32(255) - hp
    return np.concatenate([np.array([theme_color(theme)], np.float32), hp])


def view_bytes(H, W):
    """Bytes of one image's two (H, W, 3) uint8 views."""
    return 2 * H * W * 3


def check(inputs, hms, hm_hps, dr):
    """Raises ValueError unless every ``inputs[i]`` is a (3, H, W), ``hms[i]`` a (1, h, w) and ``hm_hps[i]`` a
    (C, h, w) contiguous float32 CUDA tensor with H = h * dr, W = w * dr and 1 <= C <= 17.  Returns the
    ``(H, W, h, w, C)`` of each image."""
    if not len(inputs) == len(hms) == len(hm_hps):
        raise ValueError("heatmaps: %d inputs, %d hm and %d hm_hp maps" % (len(inputs), len(hms), len(hm_hps)))
    if len(inputs) > 65535:
        raise ValueError("heatmaps: %d images exceed one launch (max 65535)" % len(inputs))
    dr = int(dr)
    if dr < 1:
        raise ValueError("heatmaps: down ratio %d" % dr)
    sizes = []
    for i, (x, hm, hp) in enumerate(zip(inputs, hms, hm_hps)):
        for name, t in (("input", x), ("hm", hm), ("hm_hp", hp)):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 3 or not t.is_contiguous():
                raise ValueError("heatmaps: %s %d must be a contiguous 3-d float32 tensor, got %s" % (
                    name, i, (t.dtype, tuple(t.shape)) if isinstance(t, torch.Tensor) else type(t).__name__))
        (c3, H, W), (c1, h, w), (C, h2, w2) = x.shape, hm.shape, hp.shape
        if c3 != 3 or c1 != 1 or not 1 <= C <= MAX_C or (h2, w2) != (h, w) or min(h, w) < 1:
            raise ValueError("heatmaps: image %d has input %s, hm %s, hm_hp %s; expected (3, H, W), (1, h, w) and "
                             "(C, h, w) with 1 <= C <= %d" % (i, tuple(x.shape), tuple(hm.shape), tuple(hp.shape), MAX_C))
        if (H, W) != (h * dr, w * dr) or H * W >= 2 ** 31:
            raise ValueError("heatmaps: image %d: a %dx%d map at down ratio %d does not make a %dx%d input"
                             % (i, h, w, dr, H, W))
        if not (x.is_cuda and hm.is_cuda and hp.is_cuda):
            raise ValueError("heatmaps: image %d is not on a CUDA device" % i)
        sizes.append((H, W, h, w, C))
    return sizes


def layout(sources, sizes, dr, out_offsets=None):
    """The launch table of images whose ``(input, hm, hm_hp)`` device addresses are ``sources`` and whose
    ``(H, W, h, w, C)`` are ``sizes``.  Each image's two views go to byte ``out_offsets[i]`` of the output (packed from
    0 without it).  Returns ``(table, out_offsets, workspace_bytes)``."""
    table = np.zeros(len(sizes), IMAGE)
    if out_offsets is None:
        out_offsets = np.cumsum([0] + [view_bytes(H, W) for H, W, _, _, _ in sizes])[:-1].tolist()
    ws = 0
    for n, ((x, hm, hp), (H, W, h, w, C), o) in enumerate(zip(sources, sizes, out_offsets)):
        table[n] = (x, hm, hp, o, ws, H, W, h, w, C, dr)
        ws += (2 * (h * w + H * W) * 3 + 15) // 16 * 16
    return table, list(out_offsets), max(ws, 16)


def launch(table, workspace_bytes, theme, mean, std, out):
    """One upload of ``table`` and one ``cpb200_heatmap_views_batch`` writing into the uint8 CUDA tensor ``out``."""
    import ctypes
    from . import _lib
    dev = out.device
    host = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).pin_memory()
    buf = host.to(dev, non_blocking=True)
    ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=dev)
    col = colors(theme).reshape(-1)
    col = (ctypes.c_float * col.size)(*col)
    mean = (ctypes.c_float * 3)(*np.asarray(mean, np.float32).reshape(-1))
    std = (ctypes.c_float * 3)(*np.asarray(std, np.float32).reshape(-1))
    with torch.cuda.device(dev):
        st = _lib.lib().cpb200_heatmap_views_batch(buf.data_ptr(), len(table), col, mean, std,
                                                   1 if theme == "white" else 0, out.data_ptr(), ws.data_ptr(),
                                                   torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(st, "heatmap_views_batch")


def download(out, offsets, shapes):
    """One device-to-host copy of the views: one ``{'pred_hm', 'pred_hmhp'}`` dict of (H, W, 3) uint8 arrays per
    image."""
    host = out.cpu().numpy()
    res = []
    for o, (H, W) in zip(offsets, shapes):
        n = H * W * 3
        res.append({VIEWS[0]: host[o:o + n].reshape(H, W, 3), VIEWS[1]: host[o + n:o + 2 * n].reshape(H, W, 3)})
    return res


def views(inputs, hms, hm_hps, dr, theme, mean, std):
    """Both views of each image: ``inputs[i]`` its normalized (3, H, W) network input, ``hms[i]`` its (1, h, w) and
    ``hm_hps[i]`` its (C, h, w) heat maps as ``process()`` leaves them, all contiguous float32 CUDA tensors;
    ``mean`` / ``std`` the normalization.  One launch table, three kernels, one copy back."""
    sizes = check(inputs, hms, hm_hps, dr)
    if not sizes:
        return []
    table, offsets, ws = layout([(x.data_ptr(), hm.data_ptr(), hp.data_ptr()) for x, hm, hp in zip(inputs, hms, hm_hps)],
                                sizes, dr)
    out = torch.empty(max(sum(view_bytes(H, W) for H, W, _, _, _ in sizes), 1), dtype=torch.uint8,
                      device=inputs[0].device)
    launch(table, ws, theme, mean, std, out)
    return download(out, offsets, [(H, W) for H, W, _, _, _ in sizes])
