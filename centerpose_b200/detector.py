"""Host-side mirror of the reference's detector classes (``lib/detectors/base_detector.py``,
``lib/detectors/multi_pose.py``, ``lib/detectors/detector_factory.py``): same constructor,
``run / pre_process / process / post_process / merge_outputs`` methods, result dictionary and the
seven timing keys — with the network forward and the decode running as fused CUDA kernels.

Differences that are additive only:
  * ``process`` hands the head logits to the decode kernel, which applies the logistic itself
    (``multi_pose.py:35-37`` folded into the kernel); the returned ``outputs`` still carry the
    sigmoid'ed ``hm`` / ``hm_hp`` like the reference's in-place ``sigmoid_``;
  * flip-test averaging (``multi_pose.py:45-53``) is done on the device — the reference's
    ``flip_lr`` / ``flip_lr_off`` round-trip through numpy (``lib/models/utils.py:30-47``);
  * ``run_batch`` (new): many pre-processed images per call — the reference API is single-image;
  * ``run_images`` (new): ``run()`` for a list of raw images, batched on the device, with the reference's
    test-time flip / multi-scale / soft-NMS settings.
"""
from __future__ import annotations

import time

import cv2
import numpy as np
import torch

from .decode import affine_for_meta, flip_merge, multi_pose_decode, sigmoid_
from .image import get_affine_transform, multi_pose_post_process
from .model import create_model, load_model
from .soft_nms import soft_nms_39, soft_nms_39_cuda

FLIP_IDX = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]   # multi_pose.py:27


class BaseDetector(object):
    def __init__(self, cfg):
        print("Creating model...")
        self.model = create_model(cfg.MODEL.NAME, cfg.MODEL.HEAD_CONV, cfg)
        if getattr(cfg.TEST, "MODEL_PATH", ""):
            self.model = load_model(self.model, cfg.TEST.MODEL_PATH)
        if not torch.cuda.is_available():
            raise RuntimeError("centerpose_b200 detectors need a CUDA device (no CPU path)")
        self.model = self.model.to(torch.device("cuda"))
        self.model.eval()
        self.mean = np.array(cfg.DATASET.MEAN, dtype=np.float32).reshape(1, 1, 3)
        self.std = np.array(cfg.DATASET.STD, dtype=np.float32).reshape(1, 1, 3)
        self.max_per_image = 100
        self.num_classes = cfg.MODEL.NUM_CLASSES
        self.scales = cfg.TEST.TEST_SCALES
        self.cfg = cfg
        self.pause = True
        if int(cfg.TEST.TOPK) > 128 or int(cfg.TEST.TOPK) < 1:
            # the fused decode kernel keeps K candidates per channel on chip (CPB200_DECODE_MAX_K, include/centerpose_b200.h);
            # the reference accepts any TOPK (lib/models/decode.py:235) — say so here instead of failing at the first image
            raise ValueError("centerpose_b200: TEST.TOPK must be in 1..128 (got %d); the reference default is 100" % int(cfg.TEST.TOPK))
        if int(cfg.MODEL.NUM_CLASSES) != 1:
            raise ValueError("centerpose_b200: multi_pose decoding supports NUM_CLASSES == 1 (COCO person), got %d" % int(cfg.MODEL.NUM_CLASSES))
        b200 = cfg.get("B200", None) if hasattr(cfg, "get") else getattr(cfg, "B200", None)
        # additive: cfg.B200.DEVICE_PREPROCESS (default on) — warp / normalise / transpose on the GPU (same values)
        self.device_preprocess = bool((b200 or {}).get("DEVICE_PREPROCESS", True)) if isinstance(b200, dict) else True

    def _pre_process_geometry(self, height, width, scale):
        """base_detector.py:33-47,59-61 — the resized size, network input size, forward ``trans_input`` and the
        c/s/out-size meta of an image of (height, width) at one test scale."""
        new_height, new_width = int(height * scale), int(width * scale)
        if self.cfg.TEST.FIX_RES:
            inp_height, inp_width = self.cfg.MODEL.INPUT_H, self.cfg.MODEL.INPUT_W
            c = np.array([new_width / 2., new_height / 2.], dtype=np.float32)
            s = max(height, width) * 1.0
        else:
            inp_height = (new_height | self.cfg.MODEL.PAD) + 1
            inp_width = (new_width | self.cfg.MODEL.PAD) + 1
            c = np.array([new_width // 2, new_height // 2], dtype=np.float32)
            s = np.array([inp_width, inp_height], dtype=np.float32)
        trans_input = get_affine_transform(c, s, 0, [inp_width, inp_height])
        meta = {"c": c, "s": s, "out_height": inp_height // self.cfg.MODEL.DOWN_RATIO,
                "out_width": inp_width // self.cfg.MODEL.DOWN_RATIO}
        return new_height, new_width, inp_height, inp_width, trans_input, meta

    def pre_process(self, image, scale, meta=None):
        """base_detector.py:32-62 — resize, centre-crop affine warp to the network input, normalise,
        HWC->CHW, optional mirrored copy; returns the (1 or 2,3,H,W) tensor and the c/s/out-size meta."""
        height, width = image.shape[0:2]
        new_height, new_width, inp_height, inp_width, trans_input, meta = self._pre_process_geometry(height, width, scale)
        if self.device_preprocess and image.dtype == np.uint8 and image.ndim == 3 and image.shape[2] == 3:
            # warp + normalise + HWC->CHW (+ mirrored copy) in one CUDA kernel, bit-exact with the cv2 / numpy lines
            # below (csrc/post.cu); a scale != 1 keeps cv2.resize on the host, as in the reference
            resized = image if (new_width, new_height) == (width, height) else cv2.resize(image, (new_width, new_height))
            return self._pre_process_device(resized, trans_input, inp_height, inp_width), meta
        resized = cv2.resize(image, (new_width, new_height))
        inp = cv2.warpAffine(resized, trans_input, (inp_width, inp_height), flags=cv2.INTER_LINEAR)
        inp = ((inp / 255. - self.mean) / self.std).astype(np.float32)
        images = inp.transpose(2, 0, 1).reshape(1, 3, inp_height, inp_width)
        if self.cfg.TEST.FLIP_TEST:
            images = np.concatenate((images, images[:, :, :, ::-1]), axis=0)
        images = torch.from_numpy(np.ascontiguousarray(images))
        return images, meta

    def _pre_process_device(self, image_u8, trans_input, inp_height, inp_width):
        import ctypes
        from . import _lib
        dev = torch.device("cuda")
        src = torch.from_numpy(np.ascontiguousarray(image_u8)).to(dev, non_blocking=True)
        flip = bool(self.cfg.TEST.FLIP_TEST)
        out = torch.empty((2 if flip else 1, 3, inp_height, inp_width), dtype=torch.float32, device=dev)
        M = (ctypes.c_double * 6)(*np.asarray(trans_input, np.float64).reshape(-1))
        mean = (ctypes.c_float * 3)(*np.asarray(self.mean, np.float32).reshape(-1))
        std = (ctypes.c_float * 3)(*np.asarray(self.std, np.float32).reshape(-1))
        with torch.cuda.device(dev):
            st = _lib.lib().cpb200_pre_process(src.data_ptr(), image_u8.shape[0], image_u8.shape[1], M, out.data_ptr(),
                                               inp_height, inp_width, mean, std, 1 if flip else 0,
                                               torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(st, "pre_process")
        return out

    def process(self, images, return_time=False):
        raise NotImplementedError

    def post_process(self, dets, meta, scale=1):
        raise NotImplementedError

    def merge_outputs(self, detections):
        raise NotImplementedError

    def debug(self, debugger, images, dets, output, scale=1):
        raise NotImplementedError

    def show_results(self, debugger, image, results):
        raise NotImplementedError

    # -- run(): orchestration + the reference's seven wall-clock timers -----------------------------
    def _load(self, source):
        """ndarray (BGR HWC uint8) | path | pre-processed dict -> (image, pre_processed dict or None)."""
        if isinstance(source, np.ndarray):
            return source, None
        if isinstance(source, str):
            image = cv2.imread(source)
            if image is None:
                raise FileNotFoundError(source)
            return image, None
        return source["image"][0].numpy(), source

    def run(self, image_or_path_or_tensor, meta=None):
        """Same contract as ``base_detector.py:79-140``: returns ``{'results': {1: rows}, 'tot', 'load', 'pre',
        'net', 'dec', 'post', 'merge'}`` (seconds, CUDA-synchronised like the reference's timers)."""
        clock = {k: 0.0 for k in ("load", "pre", "net", "dec", "post", "merge", "tot")}
        sync = torch.cuda.synchronize
        t_start = time.time()
        image, prepared = self._load(image_or_path_or_tensor)
        t_prev = time.time()
        clock["load"] = t_prev - t_start
        per_scale = []
        for scale in self.scales:
            if prepared is None:
                images, meta = self.pre_process(image, scale, meta)
            else:
                images = prepared["images"][scale][0]
                meta = {k: v.numpy()[0] for k, v in prepared["meta"][scale].items()}
            images = images.to(torch.device("cuda"))
            sync()
            t_now = time.time(); clock["pre"] += t_now - t_prev; t_prev = t_now
            output, dets, t_forward = self.process(images, return_time=True)
            sync()
            clock["net"] += t_forward - t_prev
            t_now = time.time(); clock["dec"] += t_now - t_forward; t_prev = t_now
            if self.cfg.DEBUG >= 2:
                self.debug(None, images, dets, output, scale)
            per_scale.append(self.post_process(dets, meta, scale))
            sync()
            t_now = time.time(); clock["post"] += t_now - t_prev; t_prev = t_now
        results = self.merge_outputs(per_scale)
        sync()
        t_end = time.time()
        clock["merge"] = t_end - t_prev
        clock["tot"] = t_end - t_start
        if self.cfg.DEBUG >= 1:
            self.show_results(None, image, results)
        out = {"results": {1: results}}
        out.update(clock)
        return out


def group_by_shape(keys, max_batch):
    """``keys[i]`` is the (scale index, input H, input W) of work item i.  Returns ``[(key, [item indices])]``: items
    with equal keys in input order, split into runs of at most ``max_batch``; groups are ordered by each key's first
    item.  Every item appears exactly once, so its results can be put back at its input position."""
    if int(max_batch) < 1:
        raise ValueError("max_batch must be >= 1, got %r" % (max_batch,))
    by_key = {}
    for i, k in enumerate(keys):
        by_key.setdefault(tuple(k), []).append(i)
    return [(k, idx[j:j + int(max_batch)]) for k, idx in by_key.items() for j in range(0, len(idx), int(max_batch))]


# one entry of cpb200_pre_process_batch's device table (struct cpb200_pre_image, include/centerpose_b200.h)
_PRE_IMAGE = np.dtype([("offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("trans_input", "<f8", (6,))])
assert _PRE_IMAGE.itemsize == 64


def _swap_pairs(C, pairs, device):
    idx = list(range(C))
    for a, b in pairs:
        idx[a], idx[b] = idx[b], idx[a]
    return torch.tensor(idx, device=device, dtype=torch.long)


class MultiPoseDetector(BaseDetector):
    def __init__(self, cfg):
        super(MultiPoseDetector, self).__init__(cfg)
        self.flip_idx = FLIP_IDX

    # -- device-side flip helpers (semantics of lib/models/utils.py:27-47 without the host round-trip)
    def _flip_lr(self, x):
        return torch.flip(x, [3]).index_select(1, _swap_pairs(x.shape[1], self.flip_idx, x.device))

    def _flip_lr_off(self, x):
        B, C, H, W = x.shape
        t = torch.flip(x, [3]).view(B, C // 2, 2, H, W).clone()
        t[:, :, 0] *= -1
        t = t.index_select(1, _swap_pairs(C // 2, self.flip_idx, x.device))
        return t.view(B, C, H, W)

    def process(self, images, return_time=False):
        """multi_pose.py:29-60."""
        cfg = self.cfg
        with torch.no_grad():
            torch.cuda.synchronize()
            outputs = self.model(images)
            hm, wh, hps, reg, hm_hp, hp_offset = outputs
            use_hm_hp = cfg.LOSS.HM_HP
            sig_hp = use_hm_hp and not cfg.LOSS.MSE_LOSS
            reg = reg if cfg.LOSS.REG_OFFSET else None
            hm_hp = hm_hp if use_hm_hp else None
            hp_offset = hp_offset if cfg.LOSS.REG_HP_OFFSET else None
            if cfg.TEST.FLIP_TEST:
                sigmoid_(hm)
                if sig_hp:
                    sigmoid_(hm_hp)
                torch.cuda.synchronize()
                forward_time = time.time()
                # one fused pass instead of ~10 torch ops (and instead of the reference's numpy round trips)
                hm, wh, hps, hm_hp = flip_merge(hm[0:2].contiguous(), wh[0:2].contiguous(), hps[0:2].contiguous(),
                                                hm_hp[0:2].contiguous() if hm_hp is not None else None, self.flip_idx)
                reg = reg[0:1] if reg is not None else None
                hp_offset = hp_offset[0:1] if hp_offset is not None else None
                dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=cfg.TEST.TOPK)
            elif sig_hp or hm_hp is None:
                # logits go straight into the decode kernel (fused logistic); `outputs` still get
                # the reference's in-place sigmoid so callers (debug viz) see the same tensors
                torch.cuda.synchronize()
                forward_time = time.time()
                dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset,
                                         K=cfg.TEST.TOPK, apply_sigmoid=True)
                sigmoid_(hm)
                if hm_hp is not None:
                    sigmoid_(hm_hp)
            else:                      # MSE_LOSS: hm_hp is used raw, hm is sigmoid'ed
                sigmoid_(hm)
                torch.cuda.synchronize()
                forward_time = time.time()
                dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=cfg.TEST.TOPK)
        if return_time:
            return outputs, dets, forward_time
        return outputs, dets

    def _decode_heads(self, outputs, affine=None):
        """Decode one forward's head maps with the cfg gating of ``process()`` (multi_pose.py:35-41): REG_OFFSET /
        REG_HP_OFFSET switch the sub-pixel offsets off, MSE_LOSS means ``hm_hp`` is used raw (no logistic), HM_HP
        must be on (the reference's decode needs the keypoint heat-maps, decode.py:307).  Leaves ``outputs`` untouched
        unless a logistic has to be applied to only one of the two heat-maps."""
        cfg = self.cfg
        hm, wh, hps, reg, hm_hp, hp_offset = outputs
        reg = reg if cfg.LOSS.REG_OFFSET else None
        hp_offset = hp_offset if cfg.LOSS.REG_HP_OFFSET else None
        if not cfg.LOSS.HM_HP:
            raise NameError("name 'hm_score' is not defined")       # what the reference raises (decode.py:307)
        if cfg.LOSS.MSE_LOSS:                                       # hm sigmoid'ed, hm_hp raw
            hm = sigmoid_(hm.clone())
            return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=cfg.TEST.TOPK, affine=affine)
        return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=cfg.TEST.TOPK,
                                 apply_sigmoid=True, affine=affine)

    def post_process(self, dets, meta, scale=1):
        """multi_pose.py:62-71 (single image: a batch is flattened into one image's rows, as there)."""
        dets = dets.detach().cpu().numpy().reshape(1, -1, dets.shape[2])
        out = multi_pose_post_process(dets.copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])
        for j in range(1, self.num_classes + 1):
            out[0][j] = np.array(out[0][j], dtype=np.float32).reshape(-1, 56)
            out[0][j][:, :4] /= scale
            out[0][j][:, 5:39] /= scale
        return out[0]

    def merge_outputs(self, detections):
        """multi_pose.py:73-79."""
        results = np.concatenate([d[1] for d in detections], axis=0).astype(np.float32)
        if self.cfg.TEST.NMS or len(self.cfg.TEST.TEST_SCALES) > 1:
            soft_nms_39(results, Nt=0.5, method=2)
        return results.tolist()

    def debug(self, debugger, images, dets, output, scale=1):
        raise NotImplementedError("visual debugging (lib/utils/debugger.py) is outside the GPU hot path")

    def show_results(self, debugger, image, results):
        raise NotImplementedError("visualisation (lib/utils/debugger.py) is outside the GPU hot path")

    # -- additive: batched / device-resident paths ------------------------------------------------
    def merge_outputs_device(self, detections, nms=None, return_keep=False):
        """Device-resident ``merge_outputs`` (multi_pose.py:73-79): ``detections`` is a list of CUDA ``(N_i, 56)``
        tensors of ONE image already in original-image pixels (one per test scale, from the fused decode +
        back-projection).  Concatenates them and, with ``TEST.NMS`` or several scales, runs ``soft_nms_39`` as ONE CUDA
        kernel (``cpb200_soft_nms_39``, pinned to the reference's compiled Cython routine).  Like the reference — which
        ignores the keep list ``soft_nms_39`` returns and hands back the WHOLE array it mutated in place (decayed scores,
        suppressed rows swapped to the tail) — this returns all rows as a CUDA ``(N, 56)`` tensor; ``return_keep=True``
        additionally returns how many leading rows survived.  No host round trip until the caller asks for numbers."""
        rows = torch.cat([d.reshape(-1, d.shape[-1]) for d in detections], dim=0).contiguous().float()
        if nms is None:
            nms = bool(self.cfg.TEST.NMS) or len(self.cfg.TEST.TEST_SCALES) > 1
        keep = rows.shape[0]
        if nms:
            keep = soft_nms_39_cuda(rows, Nt=0.5, method=2)
        return (rows, keep) if return_keep else rows

    @torch.no_grad()
    def run_batch(self, images: torch.Tensor, metas=None):
        """images (B,3,H,W) pre-processed (host or device).  Returns the (B,K,56) detections in
        output-grid units on the device, or per-image post-processed dicts when ``metas`` is given."""
        images = images.to(torch.device("cuda"), non_blocking=True)
        dets = self._decode_heads(self.model(images))
        if metas is None:
            return dets
        host = dets.cpu().numpy()
        return [self.post_process(torch.from_numpy(host[i:i + 1]), metas[i]) for i in range(host.shape[0])]

    @torch.no_grad()
    def run_batch_fused(self, images: torch.Tensor, metas, scale=1.0, nms=None):
        """Like ``run_batch(images, metas)`` but with ``post_process`` fused into the decode kernel: returns a
        ``(B, K, 56)`` float32 numpy array already in original-image pixels (one D2H copy, no host math).  With
        ``TEST.NMS`` (or ``nms=True``) every image's rows additionally go through the CUDA ``soft_nms_39`` on the
        device (multi_pose.py:73-79: rows re-ordered / scores decayed in place, all K rows returned as the reference does)."""
        from .decode import affine_for_meta
        images = images.to(torch.device("cuda"), non_blocking=True)
        aff = affine_for_meta(metas, scale).to(images.device, non_blocking=True)
        dets = self._decode_heads(self.model(images), affine=aff)
        if nms is None:
            nms = bool(self.cfg.TEST.NMS)
        if nms:
            for i in range(dets.shape[0]):
                soft_nms_39_cuda(dets[i], Nt=0.5, method=2)          # in place on the image's (K, 56) rows
        return dets.cpu().numpy()

    @torch.no_grad()
    def run_multiscale_fused(self, image):
        """Additive: the multi-scale test of ``run()`` (base_detector.py:99-127 with ``TEST_SCALES [1, 2]``-style
        configs, experiments/hrnet_w32_512.yaml:142) kept on the device end to end; ``run_images([image])[0]``.
        Returns the merged ``(N, 56)`` rows (numpy) in original-image pixels, like ``run()['results'][1]``."""
        return self.run_images([image])[0]

    @torch.no_grad()
    def run_images(self, images, max_batch=32):
        """Additive: ``run()`` for many images at once, with the reference's test-time settings (``FLIP_TEST``,
        ``TEST_SCALES``, ``FIX_RES``, ``NMS``; what tools/evaluate.py runs).  ``images`` is a list of BGR uint8 HWC
        arrays or image paths.  Returns one float32 ``(N_i, 56)`` array per image, in input order, equal to
        ``run(image)['results'][1]``: all rows, suppressed ones at the tail, as the reference's ``merge_outputs``.

        Per test scale every image gets ``pre_process``'s geometry (a scale != 1 keeps ``cv2.resize`` on the host).
        Images with the same (scale, input size) are batched, at most ``max_batch`` per forward (2x that many
        network images with ``FLIP_TEST``): one pinned upload, one ``cpb200_pre_process_batch``, the forward, the
        flip merge and the decode with the back-projection fused.  The per-scale rows are then concatenated per image
        and, with ``TEST.NMS`` or several scales, go through one ``cpb200_soft_nms_39_batch`` for all images.  The
        only host wait is the final device-to-host copy."""
        import ctypes
        from . import _lib
        from .soft_nms import soft_nms_39_cuda_batch
        if int(max_batch) < 1:
            raise ValueError("run_images: max_batch must be >= 1, got %r" % (max_batch,))
        loaded = []
        for n, src in enumerate(images):
            if not isinstance(src, (np.ndarray, str)):
                raise ValueError("run_images: image %d is a %s, expected a BGR uint8 HWC array or a path"
                                 % (n, type(src).__name__))
            image = self._load(src)[0]
            if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
                raise ValueError("run_images: image %d must be uint8 (H, W, 3), got %s %s" % (n, image.dtype, image.shape))
            loaded.append(image)
        if not loaded:
            return []
        cfg = self.cfg
        dev = torch.device("cuda")
        stream = torch.cuda.current_stream(dev).cuda_stream
        flip = bool(cfg.TEST.FLIP_TEST)
        K, S = int(cfg.TEST.TOPK), len(self.scales)
        mean = (ctypes.c_float * 3)(*np.asarray(self.mean, np.float32).reshape(-1))
        std = (ctypes.c_float * 3)(*np.asarray(self.std, np.float32).reshape(-1))
        items, keys = [], []                     # one item per (image, scale)
        for i, image in enumerate(loaded):
            height, width = image.shape[0:2]
            for si, scale in enumerate(self.scales):
                new_h, new_w, inp_h, inp_w, trans_input, meta = self._pre_process_geometry(height, width, scale)
                resized = image if (new_w, new_h) == (width, height) else cv2.resize(image, (new_w, new_h))
                items.append((i, np.ascontiguousarray(resized), trans_input, meta))
                keys.append((si, inp_h, inp_w))
        rows = torch.empty((len(loaded), S * K, 56), dtype=torch.float32, device=dev)
        for (si, inp_h, inp_w), idx in group_by_shape(keys, max_batch):
            B = len(idx)
            # one pinned buffer, one upload: [table (B x 64 B) | affine (B x 6 fp32) | image index (B int64) | pixels]
            o_aff = B * _PRE_IMAGE.itemsize
            o_idx = o_aff + B * 24 + (8 - B * 24 % 8) % 8
            o_img = o_idx + B * 8
            o_img += (16 - o_img % 16) % 16
            sizes = [items[j][1].nbytes for j in idx]
            host = torch.empty(o_img + sum(sizes), dtype=torch.uint8, pin_memory=True)
            hv = host.numpy()
            table = np.zeros(B, _PRE_IMAGE)
            pos = 0
            for n, j in enumerate(idx):
                img = items[j][1]
                table[n] = (pos, img.shape[0], img.shape[1], np.asarray(items[j][2], np.float64).reshape(6))
                hv[o_img + pos:o_img + pos + img.nbytes] = img.reshape(-1)
                pos += img.nbytes
            hv[:o_aff] = table.view(np.uint8)
            hv[o_aff:o_aff + B * 24] = affine_for_meta([items[j][3] for j in idx], self.scales[si]).numpy().view(np.uint8).reshape(-1)
            hv[o_idx:o_idx + B * 8] = np.array([items[j][0] for j in idx], np.int64).view(np.uint8)
            buf = host.to(dev, non_blocking=True)
            aff = buf[o_aff:o_aff + B * 24].view(torch.float32).view(B, 6)
            dst = buf[o_idx:o_idx + B * 8].view(torch.int64)
            inp = torch.empty((2 * B if flip else B, 3, inp_h, inp_w), dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                st = _lib.lib().cpb200_pre_process_batch(buf.data_ptr() + o_img, buf.data_ptr(), B, inp.data_ptr(),
                                                         inp_h, inp_w, mean, std, 1 if flip else 0, stream)
            _lib.check(st, "pre_process_batch")
            outputs = self.model(inp)
            if flip:
                # process()'s gating (multi_pose.py:35-53) on B [image, mirror] pairs
                hm, wh, hps, reg, hm_hp, hp_offset = outputs
                sigmoid_(hm)
                if cfg.LOSS.HM_HP and not cfg.LOSS.MSE_LOSS:
                    sigmoid_(hm_hp)
                hm, wh, hps, hm_hp = flip_merge(hm, wh, hps, hm_hp if cfg.LOSS.HM_HP else None, self.flip_idx)
                reg = reg[0::2].contiguous() if cfg.LOSS.REG_OFFSET else None
                hp_offset = hp_offset[0::2].contiguous() if cfg.LOSS.REG_HP_OFFSET else None
                dets = multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=K, affine=aff)
            else:
                dets = self._decode_heads(outputs, affine=aff)
            rows[dst, si * K:(si + 1) * K] = dets
        if cfg.TEST.NMS or S > 1:
            soft_nms_39_cuda_batch(rows, Nt=0.5, method=2)
        out = rows.cpu().numpy()
        return [out[i] for i in range(len(loaded))]


detector_factory = {"multi_pose": MultiPoseDetector}     # detector_factory.py:5-7
