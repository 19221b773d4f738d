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
    test-time flip / multi-scale / soft-NMS settings, and optionally the drawn images and the heat-map views;
  * ``run_video`` (new): tools/demo.py's video and webcam loop as a generator of per-frame rows (and drawn frames),
    frames read on a background thread (``video.FrameReader``) and batched through ``run_images``' kernels;
  * ``show_results`` / ``render_poses`` draw the detections on the device (csrc/render.cu), and ``debug()`` (DEBUG >= 2)
    blends the predicted heat maps onto the network input on the device (csrc/heatmaps.cu), byte for byte as the
    reference's Debugger.  ``debug()`` reads ``output[0]`` / ``output[4]`` and ``cfg.LOSS.HM_HP`` where the
    reference's ``output['hm']`` / ``self.LOSS.HM_HP`` would raise (INTEGRATION.md).
"""
from __future__ import annotations

import ctypes
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
        self.debug_imgs = {}        # the Debugger's imgs: what DEBUG >= 1 shows, refilled by every run()
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
            # resize, then warp + normalise + HWC->CHW (+ mirrored copy), as CUDA kernels bit-exact with the cv2 / numpy
            # lines below (csrc/post.cu), on a group of one image
            group = DeviceGroup([image], [(new_height, new_width)], [trans_input], np.zeros((1, 6), np.float32), [0])
            return group.pre_process(None, 1, (inp_height, inp_width), *self._mean_std(),
                                     bool(self.cfg.TEST.FLIP_TEST)), meta
        resized = cv2.resize(image, (new_width, new_height))
        inp = cv2.warpAffine(resized, trans_input, (inp_width, inp_height), flags=cv2.INTER_LINEAR)
        inp = ((inp / 255. - self.mean) / self.std).astype(np.float32)
        images = inp.transpose(2, 0, 1).reshape(1, 3, inp_height, inp_width)
        if self.cfg.TEST.FLIP_TEST:
            images = np.concatenate((images, images[:, :, :, ::-1]), axis=0)
        images = torch.from_numpy(np.ascontiguousarray(images))
        return images, meta

    def _mean_std(self):
        """``self.mean`` and ``self.std`` as the float[3] arrays the pre-process kernels take."""
        return tuple((ctypes.c_float * 3)(*np.asarray(v, np.float32).reshape(-1)) for v in (self.mean, self.std))

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
        self.debug_imgs = {}        # the reference makes a new Debugger per call
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
# one entry of cpb200_resize_linear_u8_batch's device table (struct cpb200_resize_image, include/centerpose_b200.h)
_RESIZE_IMAGE = np.dtype([("src_offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("dst_offset", "<i8"), ("new_h", "<i4"),
                          ("new_w", "<i4")])
assert _RESIZE_IMAGE.itemsize == 32


def resize_table(shapes, new_shapes):
    """The ``cpb200_resize_linear_u8_batch`` table that resizes HWC uint8 BGR images of ``shapes`` (h, w), packed back
    to back, to ``new_shapes`` (h, w), packed back to back in the destination.  The kernel trusts the table, so the
    sizes are checked here: each must be at least 1 and each image below 2^31 pixels."""
    table = np.zeros(len(shapes), _RESIZE_IMAGE)
    src = dst = 0
    for n, ((h, w), (new_h, new_w)) in enumerate(zip(shapes, new_shapes)):
        if min(h, w, new_h, new_w) < 1 or max(h * w, new_h * new_w) >= 2 ** 31:
            raise ValueError("resize: cannot resize a %dx%d image to %dx%d" % (h, w, new_h, new_w))
        table[n] = (src, h, w, dst, new_h, new_w)
        src += h * w * 3
        dst += new_h * new_w * 3
    return table


def pack_group(images, new_shapes, trans_inputs, affine, dst_index, alloc=lambda n: np.empty(n, np.uint8),
               src_offsets=None):
    """Lays out one upload of a ``run_images`` group of B images: ``[pre-process table (B x 64 B) | resize table
    (B x 32 B) | back-projection affines (B x 6 fp32) | destination image index (B int64) | raw pixels]``.

    ``images`` are the raw HWC uint8 images, ``new_shapes`` their (h, w) at the group's scale, ``trans_inputs`` their
    forward 2x3 warp matrices, ``affine`` the (B, 6) float32 back-projections and ``dst_index`` where each image's rows
    go.  When a size changes, the resize table sends every image into a scratch buffer of ``scratch`` bytes and the
    pre-process table reads the resized images there; otherwise there is no resize table and the pre-process table
    reads the raw pixels.  ``alloc(nbytes)`` returns the uint8 host buffer (a numpy array or a CPU tensor, e.g. pinned).
    Returns ``(buffer, layout)``; ``layout`` holds the byte offsets ``o_rsz`` (None without a resize), ``o_aff``,
    ``o_idx``, ``o_img`` and ``scratch``.

    With ``src_offsets``, the images already lie in one device buffer at those byte offsets: the tables read them
    there, ``images`` only need a ``shape``, and the buffer ends at ``o_img`` with no pixel section."""
    B = len(images)
    shapes = [im.shape[0:2] for im in images]
    resize = any(tuple(s) != tuple(n) for s, n in zip(shapes, new_shapes))
    pre = np.zeros(B, _PRE_IMAGE)
    rsz = resize_table(shapes, new_shapes) if resize else None
    if resize and src_offsets is not None:
        rsz["src_offset"] = src_offsets
    pos = 0
    for n, im in enumerate(images):
        (h, w), off = (new_shapes[n], rsz[n]["dst_offset"]) if resize else \
            (shapes[n], pos if src_offsets is None else src_offsets[n])
        pre[n] = (off, h, w, np.asarray(trans_inputs[n], np.float64).reshape(6))
        pos += im.nbytes if src_offsets is None else 0
    o_rsz = pre.nbytes if resize else None
    o_aff = pre.nbytes + (rsz.nbytes if resize else 0)
    o_idx = o_aff + B * 24                                       # B * 24 keeps the int64 index 8-byte aligned
    o_img = o_idx + B * 8
    o_img += (16 - o_img % 16) % 16
    buf = alloc(o_img + (0 if src_offsets is not None else sum(im.nbytes for im in images)))
    hv = buf.numpy() if isinstance(buf, torch.Tensor) else buf
    hv[:pre.nbytes] = pre.view(np.uint8)
    if resize:
        hv[o_rsz:o_aff] = rsz.view(np.uint8)
    hv[o_aff:o_idx] = np.ascontiguousarray(affine, np.float32).view(np.uint8).reshape(-1)
    hv[o_idx:o_idx + B * 8] = np.asarray(dst_index, np.int64).view(np.uint8)
    pos = o_img
    for im in images if src_offsets is None else ():
        hv[pos:pos + im.nbytes] = np.ascontiguousarray(im).reshape(-1)
        pos += im.nbytes
    scratch = sum(h * w * 3 for h, w in new_shapes) if resize else 0
    return buf, {"o_rsz": o_rsz, "o_aff": o_aff, "o_idx": o_idx, "o_img": o_img, "scratch": scratch}


class DeviceGroup:
    """A ``pack_group`` upload on the device and the launches that read it; it takes what ``pack_group`` takes.  The
    pinned buffer goes up without a wait on the current stream.  ``aff`` (B x 6 float32) and ``dst`` (B int64) are the
    back-projections and destination indices, views into the upload; ``scratch`` is the device buffer the resized
    images go to when a size changes, else None."""

    def __init__(self, images, new_shapes, trans_inputs, affine, dst_index, src_offsets=None):
        dev = torch.device("cuda")
        host, at = pack_group(images, new_shapes, trans_inputs, affine, dst_index,
                              alloc=lambda n: torch.empty(n, dtype=torch.uint8, pin_memory=True),
                              src_offsets=src_offsets)
        B = len(images)
        self.buf = host.to(dev, non_blocking=True)
        self.aff = self.buf[at["o_aff"]:at["o_aff"] + B * 24].view(torch.float32).view(B, 6)
        self.dst = self.buf[at["o_idx"]:at["o_idx"] + B * 8].view(torch.int64)
        self.o_rsz, self.o_img = at["o_rsz"], at["o_img"]
        self.scratch = torch.empty(at["scratch"], dtype=torch.uint8, device=dev) if at["o_rsz"] is not None else None

    def pre_process(self, pixels, B, size, mean, std, flip, f32=False):
        """Enqueues, for the group's first ``B`` images, ``cpb200_resize_linear_u8_batch`` into ``scratch`` when there
        is a resize table, then ``cpb200_pre_process_batch`` into the network input, which it returns: (B, 3, H, W)
        float32 for ``size`` (H, W), or (2B, ...) with each image's mirrored copy after it with ``flip``.  ``pixels`` is
        the device buffer ``src_offsets`` point into, or None for the pixels packed into the upload; ``mean`` and
        ``std`` are float[3].  ``f32`` normalises as the training dataset does (``cpb200_pre_process_batch_f32``,
        which makes no mirrored copy: ``flip`` must be off)."""
        from . import _lib
        dev = self.buf.device
        if pixels is None:
            pixels = self.buf.data_ptr() + self.o_img
        if self.scratch is not None:
            _lib.launch("resize_linear_u8_batch", dev, pixels, self.buf.data_ptr() + self.o_rsz, B, self.scratch)
            pixels = self.scratch
        inp = torch.empty((2 * B if flip else B, 3) + tuple(size), dtype=torch.float32, device=dev)
        if f32:
            _lib.launch("pre_process_batch_f32", dev, pixels, self.buf, B, inp, *size, mean, std)
        else:
            _lib.launch("pre_process_batch", dev, pixels, self.buf, B, inp, *size, mean, std, 1 if flip else 0)
        return inp


# run_images decodes JPEG, PNG and WebP files on the device in launches of at most this many images, whose workspace
# (JPEG coefficients and planes, PNG scanlines, WebP coefficients and planes, lossless WebP ARGB planes and prefix
# codes; reused from launch to launch) stays below
# JPEG_CHUNK_WORKSPACE bytes unless one image needs more
JPEG_CHUNK_IMAGES = 256
JPEG_CHUNK_WORKSPACE = 512 << 20
# PNG files go to the device only when a call holds at least this many of them.  The inflate is serial within a file,
# so a launch takes about as long for one file as for 256 (141-165 ms for 640x480 files on one H100), while
# cv2.imread takes 9-17 ms per file on one host thread; below this count the host decode is faster
# (tools/bench_png.py)
PNG_DEVICE_MIN_IMAGES = 16
# Lossy WebP files likewise go to the device only from this many per call on.  The entropy decode is serial within a
# file, so one launch takes about as long for one file as for 256 (51-59 ms at quality 75, 128-136 ms at 95, 640x480
# files on one H100).  run_images from quality-75 files with the device decode against cv2.imread: 0.30x for one file,
# 1.03x for 8, 1.6x for 16, 3.0x for 256 (tools/bench_webp.py)
WEBP_DEVICE_MIN_IMAGES = 16
# Lossless WebP files likewise go to the device only from this many per call on.  One launch takes 135-158 ms whether
# it holds one 640x480 file or 256 (cv2.imencode defaults, one H100).  run_images with the device decode against
# cv2.imread: 0.11x for one file, 1.0x for 16, 1.34x for 24, 1.9x for 48, 2.9x for 256 (tools/bench_webp.py --lossless)
WEBP_LOSSLESS_DEVICE_MIN_IMAGES = 24


def load_checked(n, src):
    """Input ``n`` of ``run_images`` as a BGR uint8 HWC array (a path through ``cv2.imread``)."""
    if not isinstance(src, (np.ndarray, str)):
        raise ValueError("run_images: image %d is a %s, expected a BGR uint8 HWC array or a path"
                         % (n, type(src).__name__))
    if isinstance(src, np.ndarray):
        image = src
    else:
        image = cv2.imread(src)
        if image is None:
            raise FileNotFoundError(src)
    if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
        raise ValueError("run_images: image %d must be uint8 (H, W, 3), got %s %s" % (n, image.dtype, image.shape))
    return image


def load_images_device(images):
    """Every input of ``run_images`` (a path or a BGR uint8 HWC array) in one device buffer of packed HWC uint8 BGR
    images.  It needs no model: ``train_data.TrainData`` loads its images with it too.  Returns ``(views, offsets,
    buffer)``: per input a (h, w, 3) view of its slot and the slot's byte offset.

    The files' headers are parsed first (``jpeg.parse``, ``png.parse``, ``webp.parse``, and
    ``webp_lossless.parse`` for the files ``webp.parse`` declines as lossless), so every size is known before any
    pixel exists.  The files the device can decode, with their tables, go up in one pinned buffer and are decoded
    by each format module's ``KERNEL`` (``cpb200_jpeg_decode_batch``, ``cpb200_png_decode_batch``,
    ``cpb200_webp_decode_batch``, ``cpb200_webp_lossless_decode_batch``) in chunks of at most ``JPEG_CHUNK_IMAGES``
    images that reuse one workspace; PNG files only when the call holds at least ``PNG_DEVICE_MIN_IMAGES`` of them,
    since one PNG launch costs about as much as a dozen host decodes, lossy WebP files from
    ``WEBP_DEVICE_MIN_IMAGES`` on and lossless ones from ``WEBP_LOSSLESS_DEVICE_MIN_IMAGES`` on.  The other files
    (``cv2.imread``) and the arrays take the host path, and
    their pixels go up in one copy into slots after the decoded ones.  One read of the decode status follows; a
    file whose compressed data the device found bad, or a lossless file over the device's prefix-code group
    budget, is read by ``cv2.imread`` and copied into its slot."""
    from . import _lib, jpeg, png, webp, webp_lossless
    dev = torch.device("cuda")
    datas, infos, host = {}, {}, {}
    for n, src in enumerate(images):
        if not isinstance(src, str):
            host[n] = load_checked(n, src)
            continue
        try:
            with open(src, "rb") as f:
                data = f.read()
        except OSError:
            raise FileNotFoundError(src)
        fmt = png if data[:8] == png.SIGNATURE else webp if webp.is_webp(data) else jpeg
        try:
            info = fmt.parse(data, src)
            if fmt is webp and info.reason.startswith("lossless"):
                fmt, info = webp_lossless, webp_lossless.parse(data, src)
        except ValueError:
            info = None
        if info is not None and (info.eligible or getattr(info, "progressive", None)):
            datas[n], infos[n] = data, (fmt, info)
        else:
            host[n] = load_checked(n, src)
    for fmt, least in ((png, PNG_DEVICE_MIN_IMAGES), (webp, WEBP_DEVICE_MIN_IMAGES),
                       (webp_lossless, WEBP_LOSSLESS_DEVICE_MIN_IMAGES)):
        files = [n for n in infos if infos[n][0] is fmt]
        if len(files) < least:
            for n in files:                               # cv2.imread is faster for a handful of these files
                del infos[n], datas[n]
                host[n] = load_checked(n, images[n])
    shape = {n: (info.oh, info.ow, 3) for n, (_, info) in infos.items()}
    shape.update({n: im.shape for n, im in host.items()})
    offsets, pos = {}, 0
    for n in list(infos) + list(host):                   # decoded slots first, then the host ones in one run
        offsets[n] = pos
        pos += int(np.prod(shape[n]))
    host_start = pos - sum(im.nbytes for im in host.values())
    pixels = torch.empty(max(pos, 1), dtype=torch.uint8, device=dev)
    # JPEG files, then PNG files, then lossy and lossless WebP files; status[k] belongs to dec[k]
    dec = [n for fmt in (jpeg, png, webp, webp_lossless) for n in infos if infos[n][0] is fmt]
    if dec:
        chunks, start, ws = [], 0, 0
        for k, n in enumerate(dec):
            fmt, info = infos[n]
            if k > start and (k - start == JPEG_CHUNK_IMAGES or ws + info.workspace_bytes() > JPEG_CHUNK_WORKSPACE
                              or fmt is not infos[dec[start]][0]):
                chunks.append((start, k)); start, ws = k, 0
            ws += info.workspace_bytes()
        chunks.append((start, len(dec)))
        packed = [infos[dec[a]][0].pack([infos[n][1] for n in dec[a:b]], [datas[n] for n in dec[a:b]],
                                        [offsets[n] for n in dec[a:b]])
                  for a, b in chunks]
        at = np.cumsum([0] + [p[0].nbytes + (-p[0].nbytes) % 16 for p in packed])
        up = torch.empty(int(at[-1]), dtype=torch.uint8, pin_memory=True)
        uv = up.numpy()
        for (b, _), o in zip(packed, at):
            uv[o:o + b.nbytes] = b
        src = up.to(dev, non_blocking=True)
        work = torch.empty(max(p[1] for p in packed), dtype=torch.uint8, device=dev)
        status = torch.empty(len(dec), dtype=torch.int32, device=dev)
        for (a, b), o in zip(chunks, at):
            _lib.launch(infos[dec[a]][0].KERNEL, dev, src.data_ptr() + int(o), src.data_ptr() + int(o), b - a, work,
                        work.numel(), pixels, status.data_ptr() + 4 * a)
    if host:
        staged = torch.empty(pos - host_start, dtype=torch.uint8, pin_memory=True)
        sv = staged.numpy()
        for n, im in host.items():
            sv[offsets[n] - host_start:offsets[n] - host_start + im.nbytes] = np.ascontiguousarray(im).reshape(-1)
        pixels[host_start:pos].copy_(staged, non_blocking=True)
    if dec:
        for k in np.flatnonzero(status.cpu().numpy()):
            n = dec[k]
            image = load_checked(n, images[n])
            if image.shape != shape[n]:
                raise RuntimeError("run_images: %s decodes to %s on the host, its header says %s"
                                   % (images[n], image.shape, shape[n]))
            pixels[offsets[n]:offsets[n] + image.nbytes].copy_(torch.from_numpy(image.reshape(-1)))
    views = [pixels[offsets[n]:offsets[n] + int(np.prod(shape[n]))].view(shape[n]) for n in range(len(images))]
    return views, [offsets[n] for n in range(len(images))], pixels


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
        """multi_pose.py:82-94: ``self.debug_imgs['pred_hm']`` and ``['pred_hmhp']``, the centre and keypoint heat maps
        of ``output`` (as ``process()`` leaves them) blended onto the de-normalized network input ``images[0]``, made
        on the device (``heatmaps.views``: one launch table, three kernels, one copy back).  ``debugger`` and
        ``dets`` are unused (the reference scales ``dets`` and then drops them).  ``HM_HP: false`` never gets here:
        the decode raises first."""
        from . import heatmaps
        self.debug_imgs.update(heatmaps.views([images[0].contiguous()], [output[0][0].contiguous()],
                                              [output[4][0].contiguous()], self.cfg.MODEL.DOWN_RATIO,
                                              self.cfg.DEBUG_THEME, self.mean, self.std)[0])

    def show_results(self, debugger, image, results):
        """multi_pose.py:96-107: draws every row above ``TEST.VIS_THRESH`` on a copy of ``image`` with the device
        renderer (``render_poses``) into ``self.debug_imgs['multi_pose']``, then shows every entry of
        ``self.debug_imgs`` in insertion order (with DEBUG >= 2 the heat-map views first) as the reference's
        ``Debugger.show_all_imgs`` does.  Without a cv2 GUI backend (opencv-python-headless) the display is skipped.
        ``debugger`` is unused (the reference passes its Debugger; ``run()`` passes None)."""
        self.debug_imgs["multi_pose"] = self.render_poses([image], [results])[0]
        try:
            for name, img in self.debug_imgs.items():
                cv2.imshow(name, img)
            if cv2.waitKey(0 if self.pause else 1) == 27:
                import sys
                sys.exit(0)
        except cv2.error:
            pass                                                  # no GUI backend in this cv2 build

    def render_poses(self, images, results):
        """Additive: the image ``show_results`` draws, for many images at once.  ``images`` are BGR uint8 HWC arrays,
        ``results[i]`` the ``(N_i, 56)`` rows of image i (as ``run_images`` returns them).  Returns one new annotated
        array per image, byte for byte the reference Debugger's ``imgs['multi_pose']`` (``DEBUG_THEME`` 'white' or
        any other theme).  One upload of the images and tables, one ``cpb200_render_poses_batch``, one copy back."""
        from . import render
        images = [load_checked(n, im) for n, im in enumerate(images)]
        if not images:
            return []
        shapes = [im.shape[:2] for im in images]
        ops = render.build(shapes, results, float(self.cfg.TEST.VIS_THRESH), self.cfg.DEBUG_THEME)
        pixels, offsets = render.launch(ops, images=images)
        return render.download(pixels, offsets, shapes)

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

    def run_eval(self, images, image_ids, gt, max_batch=32):
        """Additive: tools/evaluate.py's loop and ``dataset.run_eval`` (coco_hp.py:97-107) in one call.  Runs
        ``run_images(images, max_batch)``, evaluates the rows of ``images[i]`` as image ``image_ids[i]`` against ``gt``
        (a ``coco_eval.KeypointEval``, or what it takes: a ``person_keypoints_*.json`` path, its dict, or an object
        with a ``.dataset`` dict) on the device, prints the summary and returns ``stats[0]`` (AP at OKS .50:.95)."""
        from .coco_eval import KeypointEval
        ev = gt if isinstance(gt, KeypointEval) else KeypointEval(gt)
        if len(image_ids) != len(images):
            raise ValueError("run_eval: %d image ids for %d images" % (len(image_ids), len(images)))
        ev.evaluate((list(image_ids), self.run_images(images, max_batch=max_batch)))
        return ev.summarize()[0]

    @torch.no_grad()
    def run_val(self, images, image_ids, gt, max_batch=32):
        """Additive: tools/train.py's validation pass, ``trainer.val`` (``BaseTrainer.run_epoch('val')`` over the val
        split's ``MultiPoseDataset``), on the device.  ``images[i]`` (a path or a BGR uint8 array, loaded as
        ``run_images`` loads them) is image ``image_ids[i]`` of ``gt`` (a ``coco_eval.KeypointEval`` or what it takes).
        Returns ``(log_dict_val, preds)`` as ``trainer.val`` does:

        * ``log_dict_val``: the seven ``MultiPoseLoss`` stats averaged over the images as ``AverageMeter`` averages
          batches of one (a float64 sum of the float32 per-image stats, in image order, over the count), and
          ``'time'``, the elapsed minutes;
        * ``preds``: ``{image_id: {1: (TOPK, 56) float32 rows}}``, every decoded row in original-image pixels as
          ``save_result`` leaves them (no threshold, no soft-NMS); ``gt.evaluate(preds)`` is ``dataset.run_eval``.

        Per batch of at most ``max_batch`` images: the dataset's warp to ``INPUT_RES`` with its float32 normalisation
        (``cpb200_pre_process_batch_f32``), the forward, the targets (``val.targets``), the loss (``val.loss``) and the
        decode with the back-projection fused; one copy of the stats and rows at the end.  ``KeypointEval.cat_img_ids``
        lists the images the reference's val split holds.  Raises ``NotImplementedError`` for the settings
        ``val.check_cfg`` refuses."""
        from . import val
        from .coco_eval import KeypointEval
        t_start = time.time()
        cfg = self.cfg
        ev = gt if isinstance(gt, KeypointEval) else KeypointEval(gt)
        val.check_cfg(cfg, ev)
        if len(image_ids) != len(images):
            raise ValueError("run_val: %d image ids for %d images" % (len(image_ids), len(images)))
        if int(max_batch) < 1:
            raise ValueError("run_val: max_batch must be >= 1, got %r" % (max_batch,))
        for i in image_ids:
            if i not in ev.gt_range:
                raise ValueError("run_val: image id %r is not in the ground truth" % (i,))
        n = len(images)
        if n == 0:
            log = {k: 0 for k in val.STATS}
            log["time"] = (time.time() - t_start) / 60.
            return log, {}
        loaded, offsets, pixels = load_images_device(images)
        dev = torch.device("cuda")
        res, R, K = int(cfg.MODEL.INPUT_RES), int(cfg.MODEL.OUTPUT_RES), int(cfg.TEST.TOPK)
        mean, std = self._mean_std()
        stats = torch.empty((n, len(val.STATS)), dtype=torch.float32, device=dev)
        rows = torch.empty((n, K, 56), dtype=torch.float32, device=dev)
        for a in range(0, n, int(max_batch)):
            idx = list(range(a, min(n, a + int(max_batch))))
            B = len(idx)
            shapes = [tuple(loaded[i].shape[0:2]) for i in idx]
            trans, metas = [], []
            for h, w in shapes:
                c, s = val.center_scale(h, w)
                trans.append(get_affine_transform(c, s, 0, [res, res]))
                metas.append({"c": c, "s": s, "out_height": R, "out_width": R})
            group = DeviceGroup([loaded[i] for i in idx], shapes, trans, affine_for_meta(metas).numpy(), idx,
                                src_offsets=[offsets[i] for i in idx])
            outputs = self.model(group.pre_process(pixels, B, (res, res), mean, std, False, f32=True))
            tg = val.targets(ev, [image_ids[i] for i in idx], shapes, cfg)
            stats[a:a + B] = val.loss(outputs, tg, cfg)
            rows[a:a + B] = self._decode_heads(outputs, affine=group.aff)
        host_stats, host_rows = stats.cpu().numpy(), rows.cpu().numpy()
        log = {}
        for j, k in enumerate(val.STATS):
            total = 0
            for v in host_stats[:, j]:
                total += float(v)
            log[k] = total / n
        log["time"] = (time.time() - t_start) / 60.
        preds = {image_ids[i]: {1: host_rows[i]} for i in range(n)}
        return log, preds

    @torch.no_grad()
    def run_images(self, images, max_batch=32, return_images=False, return_heatmaps=False, encode_png=False):
        """Additive: ``run()`` for many images at once, with the reference's test-time settings (``FLIP_TEST``,
        ``TEST_SCALES``, ``FIX_RES``, ``NMS``; what tools/evaluate.py runs).  ``images`` is a list of BGR uint8 HWC
        arrays or image paths.  Returns one float32 ``(N_i, 56)`` array per image, in input order, equal to
        ``run(image)['results'][1]``: all rows, suppressed ones at the tail, as the reference's ``merge_outputs``.

        Per test scale every image gets ``pre_process``'s geometry.  Images with the same (scale, input size) are
        batched, at most ``max_batch`` per forward (2x that many network images with ``FLIP_TEST``).  Each batch is one
        ``DeviceGroup``: one pinned upload of its tables and raw images, at a scale != 1 one
        ``cpb200_resize_linear_u8_batch`` (``cv2.resize`` on the device, bit for bit) and one
        ``cpb200_pre_process_batch``; then the forward, the flip merge and the decode with the back-projection
        fused.  The per-scale rows are then concatenated per image
        and, with ``TEST.NMS`` or several scales, go through one ``cpb200_soft_nms_39_batch`` for all images.  The
        only host wait is the final device-to-host copy.

        With ``B200.DEVICE_PREPROCESS`` on (the default) and any path among the inputs, the images are decoded into
        one device buffer first (``load_images_device``): sequential- and progressive-Huffman JPEG files by
        ``cpb200_jpeg_decode_batch``, from ``PNG_DEVICE_MIN_IMAGES`` PNG files per call on, PNG files (not APNG)
        by ``cpb200_png_decode_batch``, from ``WEBP_DEVICE_MIN_IMAGES`` on, lossy WebP files (not alpha or animated
        ones) by ``cpb200_webp_decode_batch``, and from ``WEBP_LOSSLESS_DEVICE_MIN_IMAGES`` on, lossless WebP files
        by ``cpb200_webp_lossless_decode_batch``, byte for byte as
        ``cv2.imread``; every other file, and every array, on the host and uploaded into its slot.  The groups then
        read that buffer in place.  That adds one small device-to-host read of the decode status.  The call then
        needs device memory for the decoded images (3 bytes per pixel) and one decode chunk's workspace (JPEG: int16
        coefficients and 8-bit planes, 4.5 bytes per pixel at 4:2:0, 9 at 4:4:4; PNG: the scanlines, 1 to 8 bytes per
        pixel; WebP: 4.6 bytes per pixel of whole macroblocks; lossless WebP: about 8.8 bytes per pixel plus 575 KB
        of prefix codes per file; at most ``JPEG_CHUNK_WORKSPACE`` bytes unless one image needs more).

        With ``return_images=True`` it returns ``(rows, drawn)``: the same rows, and per image the ``render_poses``
        image of its rows (what ``show_results`` draws).  The images are then all in one device buffer (the decoded
        files where the device decode put them, the arrays uploaded once into slots after them), the groups read them
        there, and ``cpb200_render_poses_batch`` draws on them in place after the rows are known, followed by one
        device-to-host copy of the drawn images.

        With ``return_heatmaps=True`` it also returns per image the ``{'pred_hm', 'pred_hmhp'}`` views ``run()`` with
        DEBUG 2 leaves in ``debug_imgs``: ``(rows, views)``, or ``(rows, drawn, views)`` with ``return_images``.  They
        come from each image's last test scale, as ``run()`` keeps the last scale's views.  Every group at that scale
        makes its images' views with one ``cpb200_heatmap_views_batch`` after its decode (the maps get ``process()``'s
        in-place logistic first), into one device buffer that one device-to-host copy brings back.

        With ``encode_png=True`` the drawn images and the views come back as PNG files, ``bytes`` equal to
        ``cv2.imencode('.png', image)[1].tobytes()`` (what the reference's ``Debugger.save_img`` writes), instead of
        arrays: one ``cpb200_png_encode_batch`` encodes them where they are on the device, and the files are copied
        back in place of the images.  It needs ``return_images`` or ``return_heatmaps``."""
        if encode_png and not (return_images or return_heatmaps):
            raise ValueError("run_images: encode_png=True needs return_images=True or return_heatmaps=True")
        from .soft_nms import soft_nms_39_cuda_batch
        if int(max_batch) < 1:
            raise ValueError("run_images: max_batch must be >= 1, got %r" % (max_batch,))
        offsets = pixels_dev = None
        if self.device_preprocess and any(isinstance(src, str) for src in images):
            loaded, offsets, pixels_dev = load_images_device(images)
        elif return_images:
            # every image in one device buffer, so that the drawing needs no second upload
            loaded, offsets, pixels_dev = load_images_device(
                [load_checked(n, src) for n, src in enumerate(images)])
        else:
            loaded = [load_checked(n, src) for n, src in enumerate(images)]
        if not loaded:
            return ([],) * (1 + bool(return_images) + bool(return_heatmaps)) if return_images or return_heatmaps else []
        cfg = self.cfg
        dev = torch.device("cuda")
        flip = bool(cfg.TEST.FLIP_TEST)
        K, S = int(cfg.TEST.TOPK), len(self.scales)
        mean, std = self._mean_std()
        items, keys = [], []                     # one item per (image, scale)
        for i, image in enumerate(loaded):
            height, width = image.shape[0:2]
            for si, scale in enumerate(self.scales):
                new_h, new_w, inp_h, inp_w, trans_input, meta = self._pre_process_geometry(height, width, scale)
                items.append((i, (new_h, new_w), trans_input, meta))
                keys.append((si, inp_h, inp_w))
        rows = torch.empty((len(loaded), S * K, 56), dtype=torch.float32, device=dev)
        if return_heatmaps:
            from . import heatmaps
            view_shapes = [keys[i * S + S - 1][1:] for i in range(len(loaded))]
            view_at = np.cumsum([0] + [heatmaps.view_bytes(H, W) for H, W in view_shapes]).tolist()
            views_dev = torch.empty(max(view_at[-1], 1), dtype=torch.uint8, device=dev)
        for (si, inp_h, inp_w), idx in group_by_shape(keys, max_batch):
            B, n_img = len(idx), [items[j][0] for j in idx]
            # one upload of the group's tables, with the raw images unless they are on the device already
            group = DeviceGroup([loaded[i] for i in n_img], [items[j][1] for j in idx], [items[j][2] for j in idx],
                                affine_for_meta([items[j][3] for j in idx], self.scales[si]).numpy(), n_img,
                                src_offsets=None if offsets is None else [offsets[i] for i in n_img])
            inp = group.pre_process(pixels_dev, B, (inp_h, inp_w), mean, std, flip)
            outputs = self.model(inp)
            dets = self._decode_outputs(outputs, group.aff)
            if not flip and return_heatmaps and si == S - 1:
                # the decode read the logits; the views take the maps as process() leaves them
                sigmoid_(outputs[0])
                if not cfg.LOSS.MSE_LOSS:
                    sigmoid_(outputs[4])
            rows[group.dst, si * K:(si + 1) * K] = dets
            if return_heatmaps and si == S - 1:
                step = 2 if flip else 1
                hm, hm_hp = outputs[0], outputs[4]
                heatmaps.check([inp[b * step] for b in range(B)], [hm[b * step] for b in range(B)],
                               [hm_hp[b * step] for b in range(B)], cfg.MODEL.DOWN_RATIO)
                table, _, ws = heatmaps.layout(
                    [(inp[b * step].data_ptr(), hm[b * step].data_ptr(), hm_hp[b * step].data_ptr()) for b in range(B)],
                    [(inp_h, inp_w, hm.shape[2], hm.shape[3], hm_hp.shape[1])] * B, cfg.MODEL.DOWN_RATIO,
                    [view_at[i] for i in n_img])
                heatmaps.launch(table, ws, cfg.DEBUG_THEME, self.mean, self.std, views_dev)
        if cfg.TEST.NMS or S > 1:
            soft_nms_39_cuda_batch(rows, Nt=0.5, method=2)
        out = rows.cpu().numpy()
        rows_out = [out[i] for i in range(len(loaded))]
        if not (return_images or return_heatmaps):
            return rows_out
        res = (rows_out,)
        if return_images:
            from . import render
            shapes = [tuple(im.shape[:2]) for im in loaded]
            ops = render.build(shapes, rows_out, float(cfg.TEST.VIS_THRESH), cfg.DEBUG_THEME)
            render.launch(ops, pixels=pixels_dev, offsets=offsets)
            if not encode_png:
                res += (render.download(pixels_dev, offsets, shapes),)
        if return_heatmaps and not encode_png:
            res += (heatmaps.download(views_dev, view_at[:-1], view_shapes),)
        if encode_png:
            # the drawn images, then each image's two views, encoded in one launch where they are
            from . import png
            at, sh = [], []
            if return_images:
                at += [pixels_dev.data_ptr() + offsets[n] for n in range(len(loaded))]
                sh += shapes
            if return_heatmaps:
                for o, (H, W) in zip(view_at[:-1], view_shapes):
                    at += [views_dev.data_ptr() + o, views_dev.data_ptr() + o + H * W * 3]
                    sh += [(H, W)] * 2
            files = png.encode_at(at, sh, [3 * w for _, w in sh], dev)
            if return_images:
                res += (files[:len(loaded)],)
                files = files[len(loaded):]
            if return_heatmaps:
                res += ([dict(zip(heatmaps.VIEWS, files[2 * i:2 * i + 2])) for i in range(len(loaded))],)
        return res

    # -- additive: video and webcam streams (tools/demo.py's video branch) --------------------------
    def run_video(self, source, max_batch=None, return_images=False, encode_png=False):
        """Additive: tools/demo.py's video and webcam loop (``detector.run(img)`` per ``cv2.VideoCapture`` frame) as a
        generator.  ``source`` is a video path, ``"webcam"``, a camera index or an iterable of BGR uint8 (H, W, 3)
        arrays (``video.FrameReader``).  Yields ``(frame_index, rows)`` in frame order, ``rows`` the float32 (N, 56)
        array ``run_images([frame])[0]`` returns, bit for bit, under the same test settings (``FLIP_TEST``,
        ``TEST_SCALES``, ``FIX_RES``, ``NMS``); like those, they match ``run(frame)['results'][1]`` up to ``run()``'s
        host back-projection.  With ``return_images=True`` it yields ``(frame_index, rows, drawn)``, ``drawn`` what
        ``render_poses([frame], [rows])`` draws, byte for byte, or with ``encode_png=True`` its PNG file as
        ``run_images`` encodes it.  The drawing tables are built on the device from the rows
        (``render.DevicePlan``, ``cpb200_render_plan_batch``); that needs ``TEST.VIS_THRESH >= 0``.

        Frames are batched, at most ``max_batch`` per forward (default 32; 1 for a camera, which would otherwise wait
        for frames that have not happened yet).  A batch holds frames of one shape; one ``DeviceGroup`` per test scale
        (the resize and pre-process tables and the back-projections) and the network plan are made once per shape.
        Per batch the frames go up on a copy stream into one of two device buffers while the previous batch computes,
        each scale's group runs its resize and pre-process on them as ``run_images``' groups do, then come the forward,
        ``cpb200_flip_merge``, the decode with the back-projection and ``cpb200_soft_nms_39_batch`` as in
        ``run_images``, and the rows come back into pinned memory
        without a wait; the generator waits for them one batch later.  With drawing, batch n's frames are drawn in
        their device buffer once batch n + 1 is enqueued and copied back into pinned memory without a wait
        (``encode_png`` waits for the files), and yielded one batch later still.  The work goes to the stream that
        is current when ``run_video`` is called.  A path that does not open raises
        ``FileNotFoundError`` here, before the first frame."""
        from .video import FrameReader, is_live
        if encode_png and not return_images:
            raise ValueError("run_video: encode_png=True needs return_images=True")
        if max_batch is None:
            max_batch = 1 if is_live(source) else 32
        if int(max_batch) < 1:
            raise ValueError("run_video: max_batch must be >= 1, got %r" % (max_batch,))
        if return_images and not float(self.cfg.TEST.VIS_THRESH) >= 0:
            raise ValueError("run_video: drawing on the device needs TEST.VIS_THRESH >= 0, got %r"
                             % (self.cfg.TEST.VIS_THRESH,))
        reader = FrameReader(source, slots=2 * int(max_batch) + 2)
        return self._video_frames(reader, int(max_batch), bool(return_images), bool(encode_png),
                                  torch.cuda.current_stream(torch.device("cuda")))

    def _video_shape(self, h, w, max_batch):
        """What every batch of (h, w) frames shares: per test scale the ``DeviceGroup`` of ``max_batch`` frames lying
        back to back in a pixel buffer and its network input size, and two such pixel buffers."""
        dev = torch.device("cuda")
        scales = []
        frame = np.broadcast_to(np.uint8(0), (h, w, 3))
        for scale in self.scales:
            new_h, new_w, inp_h, inp_w, trans_input, meta = self._pre_process_geometry(h, w, scale)
            aff = affine_for_meta([meta], scale).numpy()
            group = DeviceGroup([frame] * max_batch, [(new_h, new_w)] * max_batch, [trans_input] * max_batch,
                                np.repeat(aff, max_batch, 0), list(range(max_batch)),
                                src_offsets=[b * h * w * 3 for b in range(max_batch)])
            scales.append((group, (inp_h, inp_w)))
        return {"hw": (h, w), "scales": scales,
                "pixels": [torch.empty(max_batch * h * w * 3, dtype=torch.uint8, device=dev) for _ in range(2)]}

    def _decode_outputs(self, outputs, aff):
        """The decode, with the back-projections ``aff``, of one forward of B images (B [image, mirror] pairs with
        ``FLIP_TEST``) for ``run_images`` and ``run_video``: ``process()``'s gating (multi_pose.py:35-53)."""
        cfg = self.cfg
        if not cfg.TEST.FLIP_TEST:
            return self._decode_heads(outputs, affine=aff)
        hm, wh, hps, reg, hm_hp, hp_offset = outputs
        sigmoid_(hm)
        if cfg.LOSS.HM_HP and not cfg.LOSS.MSE_LOSS:
            sigmoid_(hm_hp)
        hm, wh, hps, hm_hp = flip_merge(hm, wh, hps, hm_hp if cfg.LOSS.HM_HP else None, self.flip_idx)
        reg = reg[0::2].contiguous() if cfg.LOSS.REG_OFFSET else None
        hp_offset = hp_offset[0::2].contiguous() if cfg.LOSS.REG_HP_OFFSET else None
        return multi_pose_decode(hm, wh, hps, reg=reg, hm_hp=hm_hp, hp_offset=hp_offset, K=int(cfg.TEST.TOPK),
                                 affine=aff)

    def _video_batch(self, shape, pix, B):
        """Enqueues one batch of B frames lying in ``pix`` on the current stream; returns its (B, S * K, 56) rows."""
        from .soft_nms import soft_nms_39_cuda_batch
        cfg = self.cfg
        K, S = int(cfg.TEST.TOPK), len(self.scales)
        mean, std = self._mean_std()
        rows = torch.empty((B, S * K, 56), dtype=torch.float32, device=pix.device)
        for si, (group, size) in enumerate(shape["scales"]):
            inp = group.pre_process(pix, B, size, mean, std, bool(cfg.TEST.FLIP_TEST))
            rows[:, si * K:(si + 1) * K] = self._decode_outputs(self.model(inp), group.aff[:B])
        if cfg.TEST.NMS or S > 1:
            soft_nms_39_cuda_batch(rows, Nt=0.5, method=2)
        return rows

    def _video_frames(self, reader, max_batch, return_images, encode_png, compute):
        """The generator of ``run_video``.  All its device work goes to ``compute`` (the caller's stream when
        ``run_video`` was called) and to its own copy stream, whatever stream is current when it resumes.  Batch n's
        upload and compute are enqueued before batch n - 1 is finished; with drawing, batch n - 1's drawing is
        enqueued then too, and its frames are yielded once batch n's is enqueued, so each wait is for work enqueued
        one batch earlier."""
        from . import render
        dev = torch.device("cuda")
        copy = torch.cuda.Stream(dev)
        plan = render.DevicePlan(self.cfg.TEST.VIS_THRESH, self.cfg.DEBUG_THEME, dev) if return_images else None
        shape = None                   # the state of the current frame shape; a new shape replaces it
        host_rows = [None, None]
        n_batch = 0
        computed = drawn = None        # the batch whose rows are on their way back; the batch being drawn

        def batches():
            batch = []
            for fr in reader:
                if batch and (fr.image.shape != batch[0].image.shape or len(batch) == max_batch):
                    yield batch
                    batch = []
                batch.append(fr)
                if len(batch) == max_batch or reader.live:
                    yield batch
                    batch = []
            if batch:
                yield batch

        def rows_of(p):
            """Waits for batch p's rows, copies them out and hands its frames back to the reader."""
            p["ready"].synchronize()
            rows = p["host"][:p["B"]].numpy()
            p["out"] = [(fr.index, rows[b].copy()) for b, fr in enumerate(p["frames"])]
            for fr in p["frames"]:
                fr.release()
            return p["out"]

        def draw(p):
            """Enqueues batch p's drawing in place in its pixel buffer and the copy of the drawn frames."""
            rows_of(p)
            h, w = p["shape"]["hw"]
            B, hw3 = p["B"], h * w * 3
            plan.draw(p["plan"], p["pix"])
            if encode_png:
                from . import png
                p["drawn"] = png.encode_at([p["pix"].data_ptr() + b * hw3 for b in range(B)], [(h, w)] * B,
                                           [3 * w] * B, dev)
            else:
                host = p["shape"]["drawn"][p["k"]]
                host[:B * hw3].copy_(p["pix"][:B * hw3], non_blocking=True)
                p["drawn_ready"] = torch.cuda.Event()
                p["drawn_ready"].record(compute)
            p["free"].record(compute)

        def drawn_of(p):
            h, w = p["shape"]["hw"]
            if encode_png:
                drawn = p["drawn"]
            else:
                p["drawn_ready"].synchronize()
                hv = p["shape"]["drawn"][p["k"]].numpy()
                drawn = [hv[b * h * w * 3:(b + 1) * h * w * 3].reshape(h, w, 3).copy() for b in range(p["B"])]
            return [(i, r, d) for (i, r), d in zip(p["out"], drawn)]

        try:
            with torch.no_grad():
                for frames in batches():
                    with torch.cuda.stream(compute):
                        B = len(frames)
                        h, w = frames[0].image.shape[:2]
                        if shape is None or shape["hw"] != (h, w):
                            shape = self._video_shape(h, w, max_batch)
                            shape["free"] = [torch.cuda.Event(), torch.cuda.Event()]
                            shape["next"] = 0
                            for t in shape["pixels"]:
                                t.record_stream(copy)
                            # the new pixel buffers can reuse memory that work already enqueued on the compute
                            # stream still uses, so the copy stream writes into them only after that work
                            copy.wait_stream(compute)
                            if return_images and not encode_png:
                                shape["drawn"] = [torch.empty(max_batch * h * w * 3, dtype=torch.uint8,
                                                              pin_memory=True) for _ in range(2)]
                        k = shape["next"]
                        shape["next"] = 1 - k
                        pix, hw3 = shape["pixels"][k], h * w * 3
                        # the upload waits until the batch before last (the last user of this buffer) is done with it
                        copy.wait_event(shape["free"][k])
                        with torch.cuda.stream(copy):
                            for b, fr in enumerate(frames):
                                pix[b * hw3:(b + 1) * hw3].copy_(fr.slot, non_blocking=True)
                            uploaded = torch.cuda.Event()
                            uploaded.record(copy)
                        compute.wait_event(uploaded)
                        rows = self._video_batch(shape, pix, B)
                        batch = {"frames": frames, "B": B, "shape": shape, "pix": pix, "k": k, "free": shape["free"][k]}
                        if return_images:
                            batch["plan"] = plan.plan(rows, h, w)
                        j = n_batch % 2
                        n_batch += 1
                        if host_rows[j] is None:
                            host_rows[j] = torch.empty((max_batch,) + tuple(rows.shape[1:]), dtype=torch.float32,
                                                       pin_memory=True)
                        host_rows[j][:B].copy_(rows, non_blocking=True)
                        batch["host"] = host_rows[j]
                        batch["ready"] = torch.cuda.Event()
                        batch["ready"].record(compute)
                        if not return_images:
                            batch["free"].record(compute)
                            out = rows_of(computed) if computed is not None else []
                        else:
                            out = drawn_of(drawn) if drawn is not None else []
                            drawn = None
                            if computed is not None:
                                draw(computed)
                                drawn = computed
                        computed = batch
                    yield from out
                with torch.cuda.stream(compute):
                    out = []
                    if return_images:
                        if drawn is not None:
                            out += drawn_of(drawn)
                        if computed is not None:
                            draw(computed)
                            out += drawn_of(computed)
                    elif computed is not None:
                        out = rows_of(computed)
                    computed = drawn = None
                yield from out
        finally:
            reader.close()
            compute.wait_stream(copy)


detector_factory = {"multi_pose": MultiPoseDetector}     # detector_factory.py:5-7
