"""Host side of the pose drawing: what ``MultiPoseDetector.show_results`` draws (the reference's
``Debugger.add_coco_bbox`` + ``add_coco_hp`` for each row above ``TEST.VIS_THRESH``) turned into the tables of
``cpb200_render_poses_batch`` (``csrc/render.cu``), which draws it on the device byte for byte as cv2 4.13 does.

Per drawn person the tables hold the int32 box, the label box sized by ``cv2.getTextSize(txt, SIMPLEX, 0.5, 2)``, the
label text as per-pixel 256-entry tables, the joints to mark and the limb polygons from ``cv2.ellipse2Poly``.  The text
tables are captured from ``cv2.putText`` on the 256 uniform grey backgrounds, once per process for each string and
each way the image border cuts the text (anti-aliasing near a border depends on where the border is).
"""
from __future__ import annotations

import math

import cv2
import numpy as np
import torch

# the COCO person skeleton the reference's Debugger draws for dataset 'coco_hp', in its order
EDGES = ((0, 1), (0, 2), (1, 3), (2, 4), (3, 5), (4, 6), (5, 6), (5, 7), (7, 9), (6, 8), (8, 10), (5, 11), (6, 12),
         (11, 12), (11, 13), (13, 15), (12, 14), (14, 16))
JOINTS = 17
# the colour (BGR) of each joint's heat map in the Debugger's 'pred_hmhp' view (its colors_hp), in joint order
JOINT_COLORS = ((255, 0, 255), (255, 0, 0), (0, 0, 255), (255, 0, 0), (0, 0, 255), (255, 0, 0), (0, 0, 255),
                (255, 0, 0), (0, 0, 255), (255, 0, 0), (0, 0, 255), (255, 0, 0), (0, 0, 255), (255, 0, 0), (0, 0, 255),
                (255, 0, 0), (0, 0, 255))
STICK_WIDTH = 2
FONT = cv2.FONT_HERSHEY_SIMPLEX
# the box and label colour of class 0 (BGR): the 'white' theme draws the inverted, clipped last colour of the
# Debugger's palette, every other theme the palette's first colour
THEME_COLORS = {"white": (255, 128, 128)}
OTHER_THEME_COLOR = (255, 255, 255)

IMAGE = np.dtype([("offset", "<i8"), ("ws_offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("person_begin", "<i4"),
                  ("person_count", "<i4"), ("limb_begin", "<i4"), ("limb_count", "<i4")])
PERSON = np.dtype([("box", "<i4", 4), ("label", "<i4", 4), ("text_x", "<i4"), ("text_y", "<i4"), ("text_begin", "<i4"),
                   ("text_count", "<i4"), ("color", "u1", 4), ("joints", "<i4"), ("limb_begin", "<i4"),
                   ("limb_count", "<i4"), ("fold_box", "<i4", 4), ("joint_x", "<i4", JOINTS), ("joint_y", "<i4", JOINTS),
                   ("pad", "<i4", 2)])
LIMB = np.dtype([("vert_begin", "<i4"), ("vert_count", "<i4"), ("row0", "<i4"), ("row1", "<i4"), ("rows_offset", "<i8")])
TEXT_PX = np.dtype([("dx", "<i2"), ("dy", "<i2"), ("lut", "<i4")])
assert (IMAGE.itemsize, PERSON.itemsize, LIMB.itemsize, TEXT_PX.itemsize) == (40, 224, 24, 8)

_TEXT_MARGIN = 4
_text_cache = {}


def theme_color(theme):
    return THEME_COLORS.get(theme, OTHER_THEME_COLOR)


def label_text(score):
    return "p{:.1f}".format(score)


def _text_extent(txt):
    """(x0, x1, y0, y1) around the origin that holds every pixel ``cv2.putText(txt, SIMPLEX, 0.5, thickness 1, LINE_AA)``
    can touch."""
    (tw, th), base = cv2.getTextSize(txt, FONT, 0.5, 1)
    m = _TEXT_MARGIN
    return -m, tw + m, -th - m, base + m


def text_table(txt, ax, bx, ay, by):
    """The pixels ``cv2.putText(img, txt, origin, SIMPLEX, 0.5, (0, 0, 0), 1, LINE_AA)`` changes when the image spans
    [ax, bx] x [ay, by] around the origin (clamped to the text's extent): ``(dx, dy, luts)``, where the pixel at
    origin + (dx, dy) becomes ``luts[k][v]`` for each channel value v.  Captured once per process from cv2."""
    key = (txt, ax, bx, ay, by)
    hit = _text_cache.get(key)
    if hit is not None:
        return hit
    h, w = by - ay + 1, bx - ax + 1
    stack = np.empty((256, h, w), np.uint8)
    for v in range(256):
        img = np.full((h, w, 3), v, np.uint8)
        cv2.putText(img, txt, (-ax, -ay), FONT, 0.5, (0, 0, 0), 1, cv2.LINE_AA)
        if not ((img[..., 0] == img[..., 1]).all() and (img[..., 0] == img[..., 2]).all()):
            raise RuntimeError("cv2.putText drew grey text in colour; the per-channel text tables do not hold")
        stack[v] = img[..., 0]
    ys, xs = np.nonzero((stack != np.arange(256, dtype=np.uint8)[:, None, None]).any(0))
    x0, x1, y0, y1 = _text_extent(txt)
    if (ax, bx, ay, by) == (x0, x1, y0, y1) and len(ys) and (ys.min() == 0 or xs.min() == 0 or ys.max() == h - 1
                                                            or xs.max() == w - 1):
        raise RuntimeError("cv2.putText drew %r past its extent" % txt)
    hit = ((xs + ax).astype(np.int16), (ys + ay).astype(np.int16), np.ascontiguousarray(stack[:, ys, xs].T))
    _text_cache[key] = hit
    return hit


def _i32(v):
    """A Python int wrapped to int32, as numpy's int32 arithmetic in the reference wraps."""
    return (int(v) + 2 ** 31) % 2 ** 32 - 2 ** 31


def limb_polygon(points, a, b):
    """The polygon the reference fills for the limb between joints a and b of the int32 (17, 2) ``points``: an
    ellipse of half-length int(length / 2) and half-width 2 around the mid-point, at int(angle) degrees.  The
    arithmetic is numpy's on int32 values (the reference names the y coordinates X and the x coordinates Y, so the
    angle is atan2 of the y difference over the x difference)."""
    ya, yb = points[a, 1], points[b, 1]
    xa, xb = points[a, 0], points[b, 0]
    dy, dx = ya - yb, xa - xb
    cy, cx = np.mean([ya, yb]), np.mean([xa, xb])
    length = (dy ** 2 + dx ** 2) ** 0.5
    angle = math.degrees(math.atan2(dy, dx))
    return cv2.ellipse2Poly((int(cx), int(cy)), (int(length / 2), STICK_WIDTH), int(angle), 0, 360, 1)


class Ops:
    """The tables of one ``cpb200_render_poses_batch`` launch (see ``build``)."""

    def __init__(self, images, persons, limbs, verts, text_px, luts, workspace_bytes):
        self.images, self.persons, self.limbs, self.verts = images, persons, limbs, verts
        self.text_px, self.luts, self.workspace_bytes = text_px, luts, workspace_bytes


def build(shapes, results, vis_thresh, theme="white"):
    """The launch tables that draw ``results[i]`` (rows of 56: box, score, 17 (x, y), 17 joint scores) on image i of
    (h, w) ``shapes[i]`` as ``show_results`` does: each row whose score is above ``vis_thresh``, in row order.  Scores
    compare as Python floats, as the list rows of ``run()`` do (so a float32 0.3 is above a threshold of 0.3)."""
    if len(shapes) != len(results):
        raise ValueError("render: %d images but %d result arrays" % (len(shapes), len(results)))
    color = theme_color(theme)
    images = np.zeros(len(shapes), IMAGE)
    persons, limbs, verts, text_px = [], [], [], []
    lut_at, luts = {}, []
    n_verts = n_text = 0
    ws = 0
    for i, ((h, w), rows) in enumerate(zip(shapes, results)):
        h, w = int(h), int(w)
        if h < 1 or w < 1:
            raise ValueError("render: image %d is %dx%d" % (i, h, w))
        rows = np.asarray(rows)
        if rows.size and (rows.ndim != 2 or rows.shape[1] != 56):
            raise ValueError("render: results[%d] must be (N, 56) rows, got %s" % (i, rows.shape))
        ws_img, ws_rows = ws, ws + (h * w + 7) // 8 * 8
        p0, l0 = len(persons), len(limbs)
        for row in rows.reshape(-1, 56):
            score = float(row[4])
            if not score > vis_thresh:
                continue
            p = np.zeros((), PERSON)
            box = np.array(row[:4], dtype=np.int32)
            txt = label_text(score)
            tw, th = cv2.getTextSize(txt, FONT, 0.5, 2)[0]
            p["box"] = box
            p["label"] = (box[0], _i32(int(box[1]) - th - 2), _i32(int(box[0]) + tw), _i32(int(box[1]) - 2))
            p["color"][:3] = color
            ox, oy = int(box[0]), _i32(int(box[1]) - 2)
            p["text_x"], p["text_y"] = ox, oy
            x0, x1, y0, y1 = _text_extent(txt)
            ax, bx, ay, by = max(-ox, x0), min(w - 1 - ox, x1), max(-oy, y0), min(h - 1 - oy, y1)
            p["text_begin"] = n_text
            if ax <= bx and ay <= by:
                dx, dy, tl = text_table(txt, ax, bx, ay, by)
                key = (txt, ax, bx, ay, by)
                if key not in lut_at:
                    lut_at[key] = sum(len(t) for t in luts) * 256
                    luts.append(tl)
                t = np.zeros(len(dx), TEXT_PX)
                t["dx"], t["dy"], t["lut"] = dx, dy, lut_at[key] + 256 * np.arange(len(dx))
                text_px.append(t)
                p["text_count"] = len(dx)
                n_text += len(dx)
            points = np.array(row[5:39], dtype=np.int32).reshape(JOINTS, 2)
            prob = np.array(row[39:56], dtype=np.float32).reshape(JOINTS)
            p["joint_x"], p["joint_y"] = points[:, 0], points[:, 1]
            p["joints"] = int(sum(1 << j for j in range(JOINTS) if prob[j] > 0.))
            p["limb_begin"] = len(limbs)
            fx0, fy0, fx1, fy1 = w, h, -1, -1
            for a, b in EDGES:
                if not (prob[a] > 0. and prob[b] > 0.):
                    continue
                poly = np.asarray(limb_polygon(points, a, b), np.int64).reshape(-1, 2)
                ymin, ymax = int(poly[:, 1].min()), int(poly[:, 1].max())
                row0, row1 = max(ymin, 0), min(ymax, h - 1)
                limbs.append((n_verts, len(poly), row0, row1, ws_rows))
                ws_rows += max(row1 - row0 + 1, 0) * 8
                verts.append(poly.astype(np.int32))
                n_verts += len(poly)
                # every pixel the polygon can cover, with a margin
                fx0, fx1 = min(fx0, int(poly[:, 0].min()) - 2), max(fx1, int(poly[:, 0].max()) + 2)
                fy0, fy1 = min(fy0, ymin - 2), max(fy1, ymax + 2)
            p["limb_count"] = len(limbs) - p["limb_begin"]
            p["fold_box"] = (max(fx0, 0), max(fy0, 0), min(fx1, w - 1), min(fy1, h - 1))
            persons.append(p)
        images[i] = (0, ws_img, h, w, p0, len(persons) - p0, l0, len(limbs) - l0)
        ws = ws_rows
    return Ops(images, np.array(persons, PERSON).reshape(-1), np.array(limbs, LIMB).reshape(-1),
               np.concatenate(verts).reshape(-1) if verts else np.zeros(0, np.int32),
               np.concatenate(text_px) if text_px else np.zeros(0, TEXT_PX),
               np.concatenate(luts).reshape(-1) if luts else np.zeros(0, np.uint8), max(ws, 8))


def launch(ops, pixels=None, offsets=None, images=None):
    """Draws ``ops`` on the device: one upload of the tables (and of ``images``, host HWC uint8 arrays, when given),
    one ``cpb200_render_poses_batch``.  Without ``images``, the images lie in the uint8 CUDA tensor ``pixels`` at byte
    ``offsets`` and are drawn there in place.  Returns ``(pixels, offsets)`` of the drawn images."""
    from . import _lib
    dev = torch.device("cuda")
    parts = [ops.images, ops.persons, ops.limbs, ops.verts, ops.text_px, ops.luts]
    at = [0]
    for a in parts:
        at.append(at[-1] + (a.nbytes + 15) // 16 * 16)
    if images is not None:
        offsets = np.cumsum([0] + [im.nbytes for im in images])[:-1].tolist()
    table = ops.images.copy()
    table["offset"] = offsets
    parts[0] = table
    o_img = at[-1]
    total = o_img + (sum(im.nbytes for im in images) if images is not None else 0)
    host = torch.empty(max(total, 16), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for a, o in zip(parts, at):
        hv[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    if images is not None:
        for im, o in zip(images, offsets):
            hv[o_img + o:o_img + o + im.nbytes] = np.ascontiguousarray(im).reshape(-1)
    buf = host.to(dev, non_blocking=True)
    if images is not None:
        pixels = buf[o_img:]
    ws = torch.empty(ops.workspace_bytes, dtype=torch.uint8, device=dev)
    base = buf.data_ptr()
    _lib.launch("render_poses_batch", dev, pixels, base + at[0], len(table), base + at[1], base + at[2], base + at[3],
                base + at[4], base + at[5], ws)
    return pixels, offsets


def download(pixels, offsets, shapes):
    """One device-to-host copy of the drawn images: one (h, w, 3) uint8 array per image."""
    end = max((o + h * w * 3 for o, (h, w) in zip(offsets, shapes)), default=0)
    host = pixels[:end].cpu().numpy()
    return [host[o:o + h * w * 3].reshape(h, w, 3) for o, (h, w) in zip(offsets, shapes)]


# -- the drawing plan built on the device (csrc/render_plan.cu, include/centerpose_b200_video.h) ------------------
LABEL = np.dtype([(n, "<i4") for n in ("tw", "th", "x0", "x1", "y0", "y1")])
KEY = np.dtype([(n, "<i4") for n in ("label", "ax", "bx", "ay", "by", "valid")])
assert (LABEL.itemsize, KEY.itemsize) == (24, 24)
LABELS = 11                                  # p0.0 .. p1.0, every score a sigmoid and the soft-NMS decay can give
_PERSON_TEXT = PERSON.fields["text_begin"][1] // 4      # text_begin, text_count: int32 words 10 and 11


def label_string(k):
    """The label of label index k >= 0: ``label_text(score)`` for every score with round(10 * score) == k."""
    return "p%d.%d" % (k // 10, k % 10)


def label_table(n):
    """The ``cpb200_render_label`` metrics of label indices 0 .. n - 1."""
    t = np.zeros(n, LABEL)
    for k in range(n):
        txt = label_string(k)
        (tw, th), _ = cv2.getTextSize(txt, FONT, 0.5, 2)
        t[k] = (tw, th) + _text_extent(txt)
    return t


class DevicePlan:
    """Draws detection rows that are on the device with no host loop over persons or limbs.
    ``cpb200_render_plan_batch`` builds ``build()``'s person, limb and vertex tables from the rows and lists each
    person's label key (label string, border cut).  One small copy brings the keys back; the text tables of keys not
    seen before are captured from ``cv2.putText`` (``text_table``) and added to a device cache, and each person's
    text_begin / text_count is pointed at its key's entry.  ``cpb200_render_poses_batch`` then draws, byte for byte as
    ``build()`` + ``launch()``.  Everything is enqueued on the current stream."""

    def __init__(self, vis_thresh, theme, device):
        vis_thresh = float(vis_thresh)
        if not vis_thresh >= 0:
            raise ValueError("render: the device drawing plan needs TEST.VIS_THRESH >= 0, got %r" % vis_thresh)
        self.vis_thresh, self.device = vis_thresh, device
        b, g, r = theme_color(theme)
        self.color = b | g << 8 | r << 16
        self._set_labels(LABELS)
        self.verts_per_image, self.rows_per_image = 1 << 14, 1 << 20
        self._keys = {}                          # key -> (text_begin, text_count) in the cache
        self._text_px, self._luts = [np.zeros(0, TEXT_PX)], [np.zeros(0, np.uint8)]
        self._n_px = self._n_lut = 0
        self._cache = None

    def _set_labels(self, n):
        self.n_labels = n
        self._labels = torch.from_numpy(label_table(n).view(np.uint8)).to(self.device)

    def plan(self, rows, h, w):
        """Enqueues the plan of the (B, N, 56) float32 CUDA ``rows`` of B (h, w) images, and the copy of its keys to
        pinned memory.  Returns the handle ``draw`` takes."""
        from . import _lib
        B, N = int(rows.shape[0]), int(rows.shape[1])
        dev = self.device
        sizes = [B * IMAGE.itemsize, B * N * PERSON.itemsize, B * N * 18 * LIMB.itemsize,
                 B * self.verts_per_image * 8, B * N * KEY.itemsize, B * 16]
        at = np.cumsum([0] + [(s + 15) // 16 * 16 for s in sizes]).tolist()
        buf = torch.empty(max(at[-1], 16), dtype=torch.uint8, device=dev)
        base = buf.data_ptr()
        _lib.launch("render_plan_batch", dev, rows, B, N, h, w, self.vis_thresh, self.color, self._labels,
                    self.n_labels, self.verts_per_image, self.rows_per_image, base + at[0], base + at[1],
                    base + at[2], base + at[3], base + at[4], base + at[5])
        host = torch.empty(at[6] - at[4], dtype=torch.uint8, pin_memory=True)
        host.copy_(buf[at[4]:at[6]], non_blocking=True)
        done = torch.cuda.Event()
        done.record(torch.cuda.current_stream(dev))
        return {"rows": rows, "B": B, "N": N, "hw": (h, w), "buf": buf, "at": at, "host": host, "done": done,
                "verts_per_image": self.verts_per_image, "rows_per_image": self.rows_per_image}

    def _text(self, key):
        """The cache entry (text_begin, text_count) of ``key`` = (label, ax, bx, ay, by), captured when new."""
        hit = self._keys.get(key)
        if hit is None:
            k, ax, bx, ay, by = key
            dx, dy, tl = text_table(label_string(k), ax, bx, ay, by)
            t = np.zeros(len(dx), TEXT_PX)
            t["dx"], t["dy"], t["lut"] = dx, dy, self._n_lut + 256 * np.arange(len(dx))
            self._text_px.append(t)
            self._luts.append(np.ascontiguousarray(tl).reshape(-1))
            hit = self._keys[key] = (self._n_px, len(dx))
            self._n_px += len(dx)
            self._n_lut += tl.size
            self._cache = None
        return hit

    def draw(self, p, pixels):
        """Waits for ``p``'s keys, then enqueues the drawing of its B images, which lie back to back in the uint8 CUDA
        tensor ``pixels``, in place."""
        from . import _lib
        p["done"].synchronize()
        B, N = p["B"], p["N"]
        at = p["at"]
        hv = p["host"].numpy()
        keys = hv[:B * N * KEY.itemsize].view(KEY).reshape(B, N)
        counts = hv[at[5] - at[4]:at[5] - at[4] + B * 16].view(np.int32).reshape(B, 4)
        status = counts[:, 3]
        if (status == 3).any():
            raise ValueError("render: a limb's squared length overflows int32 (the reference's numpy length is NaN)")
        if (status == 2).any():
            labels = [int(keys[b, i]["label"]) for b in np.flatnonzero(status == 2) for i in range(N)]
            if min(labels) < 0 or not np.isfinite(p["rows"][..., 4].float().cpu().numpy()).all():
                raise ValueError("render: a drawn row's score is not finite")
        if (status != 0).any():
            # a vertex or span-row share, or the label table, was too small: plan again with enough of each
            need_v, need_r = int(counts[:, 1].max()), int(counts[:, 2].max())
            self.verts_per_image = max(self.verts_per_image, 1 << max(need_v - 1, 1).bit_length())
            self.rows_per_image = max(self.rows_per_image, 1 << max(need_r - 1, 1).bit_length())
            if (status == 2).any():
                scores = p["rows"][..., 4].double().cpu().numpy()
                scores = scores[scores > self.vis_thresh]
                self._set_labels(max(self.n_labels, int(np.floor(scores.max() * 10 + 1)) + 2))
            return self.draw(self.plan(p["rows"], *p["hw"]), pixels)
        n = counts[:, 0]
        text = np.zeros((B, N, 2), np.int32)
        for b in range(B):
            kb = keys[b, :n[b]]
            valid = kb["valid"] != 0
            if not valid.any():
                continue
            k5 = np.stack([kb[f] for f in ("label", "ax", "bx", "ay", "by")], 1)[valid]
            uniq, inv = np.unique(k5, axis=0, return_inverse=True)
            entries = np.array([self._text(tuple(int(v) for v in u)) for u in uniq], np.int32).reshape(-1, 2)
            text[b, np.flatnonzero(valid)] = entries[inv.reshape(-1)]
        dev = self.device
        if self._cache is None:
            px = np.concatenate(self._text_px)
            luts = np.concatenate(self._luts)
            self._cache = (torch.from_numpy(np.concatenate([px.view(np.uint8), np.zeros(16, np.uint8)])).to(dev),
                           torch.from_numpy(np.concatenate([luts, np.zeros(16, np.uint8)])).to(dev))
        buf = p["buf"]
        persons = buf[at[1]:at[1] + B * N * PERSON.itemsize].view(torch.int32).view(B * N, PERSON.itemsize // 4)
        persons[:, _PERSON_TEXT:_PERSON_TEXT + 2] = torch.from_numpy(text.reshape(-1, 2)).to(dev)
        h, w = p["hw"]
        ws = torch.empty(max(B * ((h * w + 7) // 8 * 8 + p["rows_per_image"]), 8), dtype=torch.uint8, device=dev)
        base = buf.data_ptr()
        _lib.launch("render_poses_batch", dev, pixels, base + at[0], B, base + at[1], base + at[2], base + at[3],
                    self._cache[0], self._cache[1], ws)
