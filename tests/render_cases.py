"""Seeded images and detection rows for the pose-drawing tests (``test_render_cpu.py``, ``test_render_gpu.py``,
``oracle/make_golden_render.py``, ``tools/bench_render.py``)."""
from __future__ import annotations

import numpy as np

LABEL_SCORES = [0.31 + 0.069 * k for k in range(10)] + [0.96]   # p0.3 .. p1.0


def image(h, w, seed):
    """A smooth seeded BGR image (noise would hide nothing, but gradients make blends visible)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = rng.integers(0, 256, 3)
    img = (base + 0.7 * xx[..., None] * rng.uniform(-1, 1, 3) + 0.5 * yy[..., None] * rng.uniform(-1, 1, 3)) % 256
    return (img + rng.integers(0, 12, (h, w, 3))).clip(0, 255).astype(np.uint8)


def rows(h, w, n, seed, spread=0.25, off=0.0):
    """``n`` (56,) rows like the decoder's on an (h, w) image: a box, a score, 17 joints around the box and their scores.
    ``off`` is the share of persons placed partly or wholly outside the image."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 56), np.float32)
    for i in range(n):
        far = rng.random() < off
        cx = rng.uniform(-0.6 * w, 1.6 * w) if far else rng.uniform(0, w)
        cy = rng.uniform(-0.6 * h, 1.6 * h) if far else rng.uniform(0, h)
        bw, bh = rng.uniform(4, spread * w + 5), rng.uniform(4, spread * h + 5)
        out[i, :4] = (cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2)
        out[i, 4] = rng.choice([rng.uniform(0.0, 1.0), rng.choice(LABEL_SCORES), 0.3, 0.29999998])   # around VIS_THRESH
        out[i, 5:39] = np.stack([rng.uniform(cx - bw / 2, cx + bw / 2, 17), rng.uniform(cy - bh / 2, cy + bh / 2, 17)],
                                1).reshape(-1)
        out[i, 39:] = rng.choice([rng.uniform(0.05, 1.0), 0.0, -0.1], 17, p=[0.8, 0.15, 0.05])
        if rng.random() < 0.2:                                        # zero-length limbs: joints on top of each other
            out[i, 5 + 2 * 6:5 + 2 * 7] = out[i, 5 + 2 * 5:5 + 2 * 6]
            out[i, 5 + 2 * 12:5 + 2 * 13] = out[i, 5 + 2 * 11:5 + 2 * 12]
    return out


def edge_rows(h, w):
    """Hand-placed persons: a label box cut by the top row, boxes past every border, a box inside out, a point box,
    a person with every joint at one pixel, and one with all joints off."""
    r = rows(h, w, 8, 7)
    r[:, 4] = 0.8
    r[0, 4] = 0.97                                           # p1.0
    r[0, :4] = (3, 5, w // 2, h // 2)                        # label box above row 0
    r[1, :4] = (-20, -30, w + 15, h + 9)                     # all four sides off the image
    r[2, :4] = (w - 3, h - 2, 6, 4)                          # inside out
    r[3, :4] = (w // 3, h // 3, w // 3, h // 3)              # a point
    r[4, 5:39] = np.tile([w / 2, h / 2], 17)                 # every joint at one pixel
    r[5, 39:] = 0.0                                          # no joints drawn
    r[6, :4] = (-w, -h, -5, -7)                              # wholly outside, label included
    r[6, 5:39] = np.tile([-3.0, h + 2.0], 17) + np.arange(34) * 0.5
    r[7, 5:39] = np.stack([np.linspace(-w, 2 * w, 17), np.linspace(2 * h, -h, 17)], 1).reshape(-1)   # limbs across it
    return r
