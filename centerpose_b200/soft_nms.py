"""Host soft-NMS over pose detections, semantics of ``soft_nms_39`` in the reference's Cython
module (``lib/external/nms.pyx:172-275``): IN-PLACE score decay (hard / linear / gaussian) on
float32 (N,56) rows ``[x1,y1,x2,y2,score, 34 kp coords, 17 kp scores]``.

Faithful to the reference's quirks because callers consume the mutated array, not the returned
``keep`` list (``lib/detectors/multi_pose.py:76-78``): columns 0..38 travel with a row when it is
moved, the 17 keypoint-score columns 39..55 never move (``nms.pyx:214-217``); a row whose score
falls below ``threshold`` gets columns 0..4 overwritten by the last live row and columns 5..38
swapped with it (``:257-268``); all arithmetic is C ``float``.
N <= 100 x scales, O(N^2) on the host exactly as in the reference.  The device version is ``cpb200_soft_nms_39``
(``csrc/post.cu``; ``detector.merge_outputs_device`` / ``run_batch_fused(nms=True)`` use it, ``run_images`` its batched
form ``cpb200_soft_nms_39_batch``); this port serves
``merge_outputs``, whose inputs are host arrays as in the reference."""
from __future__ import annotations

import numpy as np

F = np.float32


def soft_nms_39(boxes: np.ndarray, sigma: float = 0.5, Nt: float = 0.3, threshold: float = 0.001, method: int = 0):
    if boxes.dtype != np.float32 or boxes.ndim != 2:
        raise ValueError("soft_nms_39 expects a float32 (N, 56) array")   # Cython buffer type check
    N = boxes.shape[0]
    sigma = F(sigma); Nt = F(Nt); threshold = F(threshold); one = F(1)
    for i in range(boxes.shape[0]):
        if i >= N:
            break
        maxpos = i + int(np.argmax(boxes[i:N, 4]))           # first maximum, like the strict '<' scan
        if maxpos != i:
            tmp = boxes[i, :39].copy(); boxes[i, :39] = boxes[maxpos, :39]; boxes[maxpos, :39] = tmp
        tx1, ty1, tx2, ty2 = boxes[i, 0], boxes[i, 1], boxes[i, 2], boxes[i, 3]
        pos = i + 1
        while pos < N:
            x1, y1, x2, y2 = boxes[pos, 0], boxes[pos, 1], boxes[pos, 2], boxes[pos, 3]
            area = (x2 - x1 + one) * (y2 - y1 + one)
            iw = min(tx2, x2) - max(tx1, x1) + one
            if iw > 0:
                ih = min(ty2, y2) - max(ty1, y1) + one
                if ih > 0:
                    ua = (tx2 - tx1 + one) * (ty2 - ty1 + one) + area - iw * ih
                    ov = iw * ih / ua
                    if method == 1:
                        weight = one - ov if ov > Nt else one
                    elif method == 2:
                        weight = F(np.exp(np.float64(-(ov * ov) / sigma)))
                    else:
                        weight = F(0) if ov > Nt else one
                    boxes[pos, 4] = weight * boxes[pos, 4]
                    if boxes[pos, 4] < threshold:
                        boxes[pos, :5] = boxes[N - 1, :5]
                        tmp = boxes[pos, 5:39].copy(); boxes[pos, 5:39] = boxes[N - 1, 5:39]; boxes[N - 1, 5:39] = tmp
                        N -= 1
                        pos -= 1
            pos += 1
    return list(range(N))


def soft_nms_39_cuda(boxes, sigma: float = 0.5, Nt: float = 0.3, threshold: float = 0.001, method: int = 0) -> int:
    """Same routine on a DEVICE tensor (``cpb200_soft_nms_39``, csrc/post.cu): ``boxes`` is a contiguous CUDA
    float32 ``(N, 56)`` tensor mutated in place exactly like the host version; returns the number of kept rows."""
    import torch
    from . import _lib
    if not (boxes.is_cuda and boxes.dtype == torch.float32 and boxes.dim() == 2 and boxes.shape[1] == 56
            and boxes.is_contiguous()):
        raise ValueError("soft_nms_39_cuda expects a contiguous CUDA float32 (N, 56) tensor")
    keep = torch.zeros(1, dtype=torch.int32, device=boxes.device)
    with torch.cuda.device(boxes.device):
        st = _lib.lib().cpb200_soft_nms_39(boxes.data_ptr(), boxes.shape[0], float(sigma), float(Nt), float(threshold),
                                           int(method), keep.data_ptr(), torch.cuda.current_stream(boxes.device).cuda_stream)
    _lib.check(st, "soft_nms_39")
    return int(keep.item())


def soft_nms_39_cuda_batch(boxes, sigma: float = 0.5, Nt: float = 0.3, threshold: float = 0.001, method: int = 0):
    """``soft_nms_39_cuda`` for B images in one launch (``cpb200_soft_nms_39_batch``): ``boxes`` is a contiguous CUDA
    float32 ``(B, N, 56)`` tensor, each image's rows mutated in place exactly like the host version.  Returns the
    ``(B,)`` int32 CUDA tensor of kept-row counts; nothing waits for the device."""
    import torch
    from . import _lib
    if not (boxes.is_cuda and boxes.dtype == torch.float32 and boxes.dim() == 3 and boxes.shape[2] == 56
            and boxes.is_contiguous()):
        raise ValueError("soft_nms_39_cuda_batch expects a contiguous CUDA float32 (B, N, 56) tensor")
    keep = torch.empty(boxes.shape[0], dtype=torch.int32, device=boxes.device)
    with torch.cuda.device(boxes.device):
        st = _lib.lib().cpb200_soft_nms_39_batch(boxes.data_ptr(), boxes.shape[0], boxes.shape[1], float(sigma), float(Nt),
                                                 float(threshold), int(method), keep.data_ptr(),
                                                 torch.cuda.current_stream(boxes.device).cuda_stream)
    _lib.check(st, "soft_nms_39_batch")
    return keep
