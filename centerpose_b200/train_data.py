"""The reference's training batches on the device: ``MultiPoseDataset.__getitem__`` for split 'train'
(``lib/datasets/multi_pose.py``) over many images per call, collated as ``default_collate`` collates them.

    tr = TrainData(cfg, "person_keypoints_train2017.json")   # or a KeypointEval
    batch = tr.batch(paths, image_ids)                        # {'input', 'hm', 'reg_mask', ...} CUDA tensors

The host draws each image's random parameters in the reference's order (crop or shift and scale, rotation, flip from
``np.random``; ``color_aug``'s shuffle from ``random``; its alphas and lighting from the object's own
``data_rng = RandomState(123)``) and builds the three matrices with ``image.get_affine_transform``.  The device does
the rest: the image decode (``detector.load_images_device``), the warp and colour augmentation
(``cpb200_train_augment_batch``, csrc/augment.cu) and the targets (``cpb200_multi_pose_targets_train_batch``,
csrc/targets.cu).  With ``np.random`` and ``random`` seeded as the reference's and a fresh ``TrainData``, the batches
equal the reference's sequence of ``__getitem__`` calls over the same images, bit for bit.
"""
from __future__ import annotations

import ctypes
import random
from fractions import Fraction

import numpy as np
import torch

from . import val
from .image import get_affine_transform

# COCOHP's PCA lighting (lib/datasets/coco_hp.py)
EIG_VAL = np.array([0.2141788, 0.01817699, 0.00341571], dtype=np.float32)
EIG_VEC = np.array([[-0.58752847, -0.69563484, 0.41340352],
                    [-0.5832747, 0.00994535, -0.81221408],
                    [-0.56089297, 0.71832671, 0.41158938]], dtype=np.float32)
MAX_S = 768                                              # cpb200_train_augment_batch's largest INPUT_RES

# one entry of the device table (struct cpb200_train_image, include/centerpose_b200.h)
TRAIN_IMAGE = np.dtype([("offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("flip", "<i4"), ("rot", "<i4"),
                        ("color", "<i4"), ("order", "<i4", (3,)), ("gt_begin", "<i4"), ("gt_count", "<i4"),
                        ("alpha", "<f4", (3,)), ("beta", "<f4", (3,)), ("light", "<f8", (3,)),
                        ("trans_input", "<f8", (6,)), ("trans_output", "<f8", (6,)), ("trans_output_rot", "<f8", (6,))])
assert TRAIN_IMAGE.itemsize == 240


def get_border(border, size):
    """``MultiPoseDataset._get_border``: the crop centre's margin, halved until it fits the image."""
    i = 1
    while size - border // i <= border // i:
        i *= 2
    return border // i


def _fma(a, b, c):
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def lighting(alpha):
    """``np.dot(eig_vec, eig_val * alpha)`` for the three float64 ``alpha``: per row
    fma(v2, w2, fma(v0, w0, v1 * w1)), the order numpy's BLAS call takes, with exact rationals so that the value does
    not depend on the machine's BLAS kernel."""
    w = EIG_VAL * np.asarray(alpha, np.float64)
    v = EIG_VEC.astype(np.float64)
    return np.array([_fma(v[r, 2], w[2], _fma(v[r, 0], w[0], float(v[r, 1]) * float(w[1]))) for r in range(3)])


def mean_plan(n):
    """The summation tree of numpy's float32 ``pairwise_sum`` over ``n`` contiguous values, in the int32 layout
    ``cpb200_train_augment_batch`` reads: ``[L, D, leaf begins (L + 1), level starts (D + 1), child slot pairs]``.
    Leaves are ranges of at most 128 values; slots 0..L-1 are the leaves and L + k internal node k; the nodes are
    ordered by height, so every node's children come before it, and the root is last."""
    if n < 8 or n % 8:
        raise ValueError("mean_plan: n = %d must be a positive multiple of 8" % n)
    leaves, nodes = [], []                       # nodes: [left ref, right ref, height]; refs ('l' | 'n', index)

    def build(lo, m):
        if m <= 128:
            leaves.append(lo)
            return ("l", len(leaves) - 1), 0
        m2 = m // 2
        m2 -= m2 % 8
        a, ha = build(lo, m2)
        b, hb = build(lo + m2, m - m2)
        nodes.append([a, b, 1 + max(ha, hb)])
        return ("n", len(nodes) - 1), nodes[-1][2]

    build(0, n)
    L = len(leaves)
    order = sorted(range(len(nodes)), key=lambda k: nodes[k][2])
    pos = {k: p for p, k in enumerate(order)}
    slot = lambda ref: ref[1] if ref[0] == "l" else L + pos[ref[1]]
    heights = [nodes[k][2] for k in order]
    D = heights[-1] if heights else 0
    starts = [sum(1 for h in heights if h < d) for d in range(1, D + 2)]
    pairs = [s for k in order for s in (slot(nodes[k][0]), slot(nodes[k][1]))]
    return np.array([L, D] + leaves + [n] + starts + pairs, np.int32)


def check_cfg(cfg, ev=None):
    """Raises ``NotImplementedError`` for the settings the device batches do not cover: those ``val.check_cfg``
    refuses, and ``DEBUG > 0`` (the reference then adds ``meta`` with ``gt_det``)."""
    val.check_cfg(cfg, ev)
    if int(cfg.DEBUG) > 0:
        raise NotImplementedError("training batches with DEBUG %r (the 'meta' / 'gt_det' entries)" % (cfg.DEBUG,))


class TrainDraws:
    """The host half of the train split: the random parameters of each image, drawn in the reference's order from
    ``np.random``, ``random`` and its own ``data_rng = np.random.RandomState(123)`` (``COCOHP._data_rng``)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.data_rng = np.random.RandomState(123)

    def draw(self, h, w):
        """One image's random parameters, drawn as ``__getitem__`` draws them for an h x w image.  Returns
        ``{'c', 's', 'rot', 'flip', 'color', 'order', 'alpha', 'light'}``; the last three only with colour."""
        d = self.cfg.DATASET
        c = np.array([w / 2., h / 2.], dtype=np.float32)
        s = max(h, w) * 1.0
        rot = 0
        if d.RANDOM_CROP:
            s = s * np.random.choice(np.arange(0.6, 1.4, 0.1))
            w_border, h_border = get_border(128, w), get_border(128, h)
            c[0] = np.random.randint(low=w_border, high=w - w_border)
            c[1] = np.random.randint(low=h_border, high=h - h_border)
        else:
            sf, cf = d.SCALE, d.SHIFT
            c[0] += s * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
            c[1] += s * np.clip(np.random.randn() * cf, -2 * cf, 2 * cf)
            s = s * np.clip(np.random.randn() * sf + 1, 1 - sf, 1 + sf)
        if np.random.random() < d.AUG_ROT:
            rf = d.ROTATE
            rot = np.clip(np.random.randn() * rf, -rf * 2, rf * 2)
        flip = False
        if np.random.random() < d.FLIP:
            flip = True
            c[0] = w - c[0] - 1
        p = {"c": c, "s": s, "rot": rot, "flip": flip, "color": not d.NO_COLOR_AUG}
        if p["color"]:
            order = [0, 1, 2]
            random.shuffle(order)                       # [brightness, contrast, saturation], shuffled
            p["order"] = order
            p["alpha"] = [1. + self.data_rng.uniform(low=-0.4, high=0.4) for _ in order]
            p["light"] = lighting(self.data_rng.normal(scale=0.1, size=(3,)))
        return p


class TrainData:
    """The train split of ``MultiPoseDataset`` over the ground truth ``gt`` (a ``coco_eval.KeypointEval`` or what it
    takes: a ``person_keypoints_*.json`` path, its dict, or an object with a ``.dataset`` dict).  Owns ``data_rng``,
    ``np.random.RandomState(123)``, as ``COCOHP`` does (``self.draws.data_rng``)."""

    def __init__(self, cfg, gt):
        from .coco_eval import KeypointEval
        self.ev = gt if isinstance(gt, KeypointEval) else KeypointEval(gt)
        check_cfg(cfg, self.ev)
        S = int(cfg.MODEL.INPUT_RES)
        if S % 4 or S > MAX_S:
            raise NotImplementedError("training batches at INPUT_RES %d (a multiple of 4 up to %d)" % (S, MAX_S))
        self.cfg = cfg
        self.draws = TrainDraws(cfg)
        self._plan = None

    def table_row(self, row, p, h, w, offset, image_id):
        """Fills one ``TRAIN_IMAGE`` entry from the parameters ``p`` of an h x w image."""
        S, R = int(self.cfg.MODEL.INPUT_RES), int(self.cfg.MODEL.OUTPUT_RES)
        row["offset"], row["h"], row["w"] = offset, h, w
        row["flip"], row["rot"], row["color"] = int(p["flip"]), int(p["rot"] != 0), int(p["color"])
        if p["color"]:
            row["order"] = p["order"]
            row["alpha"] = [np.float32(a) for a in p["alpha"]]
            row["beta"] = [np.float32(1 - a) for a in p["alpha"]]
            row["light"] = p["light"]
        row["gt_begin"], row["gt_count"] = self.ev.gt_range[image_id]
        c, s, rot = p["c"], p["s"], p["rot"]
        row["trans_input"] = np.asarray(get_affine_transform(c, s, rot, [S, S]), np.float64).reshape(6)
        row["trans_output"] = np.asarray(get_affine_transform(c, s, 0, [R, R]), np.float64).reshape(6)
        row["trans_output_rot"] = np.asarray(get_affine_transform(c, s, rot, [R, R]), np.float64).reshape(6)

    def batch(self, images, image_ids):
        """``default_collate([__getitem__(i) for i in ...])`` for ``images[n]`` (a path or a BGR uint8 array, loaded as
        ``run_images`` loads them) as image ``image_ids[n]`` of the ground truth: a dict of CUDA tensors under the
        reference's keys and dtypes, ``input`` (B, 3, S, S) float32 first, then the targets, with ``reg``, ``hm_hp``
        and ``hp_offset`` / ``hp_ind`` / ``hp_mask`` present as LOSS.REG_OFFSET, HM_HP and REG_HP_OFFSET say."""
        from . import _lib
        from .detector import load_images_device
        cfg, ev = self.cfg, self.ev
        if len(images) != len(image_ids):
            raise ValueError("TrainData.batch: %d image ids for %d images" % (len(image_ids), len(images)))
        for i in image_ids:
            if i not in ev.gt_range:
                raise ValueError("TrainData.batch: image id %r is not in the ground truth" % (i,))
        B = len(images)
        if B == 0:
            raise ValueError("TrainData.batch: no images")
        S, R = int(cfg.MODEL.INPUT_RES), int(cfg.MODEL.OUTPUT_RES)
        loaded, offsets, pixels = load_images_device(images)
        dev = pixels.device
        host = torch.empty(B * TRAIN_IMAGE.itemsize, dtype=torch.uint8, pin_memory=True)
        table = host.numpy().view(TRAIN_IMAGE)
        table[:] = np.zeros(B, TRAIN_IMAGE)
        for n in range(B):
            h, w = loaded[n].shape[0:2]
            self.table_row(table[n], self.draws.draw(h, w), h, w, offsets[n], image_ids[n])
        up = host.to(dev, non_blocking=True)
        if self._plan is None or self._plan.device != dev:
            self._plan = torch.from_numpy(mean_plan(S * S)).to(dev)
        inp = torch.empty((B, 3, S, S), dtype=torch.float32, device=dev)
        ws = torch.empty(_lib.lib().cpb200_train_augment_workspace_bytes(B, S), dtype=torch.uint8, device=dev)
        mean = (ctypes.c_float * 3)(*np.asarray(cfg.DATASET.MEAN, np.float32))
        std = (ctypes.c_float * 3)(*np.asarray(cfg.DATASET.STD, np.float32))
        tg = {name: torch.empty((B,) + shape(R), dtype=dt, device=dev) for name, dt, shape in val.TARGETS}
        _lib.launch("train_augment_batch", dev, pixels, up, B, S, self._plan, mean, std, inp, ws, ws.numel())
        _lib.launch("multi_pose_targets_train_batch", dev, up, B, ev.gts, R, val.targets_struct(tg))
        out = {"input": inp}
        for k in ("hm", "reg_mask", "ind", "wh", "hps", "hps_mask"):
            out[k] = tg[k]
        if cfg.LOSS.REG_OFFSET:
            out["reg"] = tg["reg"]
        if cfg.LOSS.HM_HP:
            out["hm_hp"] = tg["hm_hp"]
        if cfg.LOSS.REG_HP_OFFSET:
            out.update({k: tg[k] for k in ("hp_offset", "hp_ind", "hp_mask")})
        return out
