"""Seeded images for the PNG encoder tests (``test_png_encode_cpu.py``, ``test_png_encode_gpu.py``,
``tools/bench_png_encode.py``).  Each case is ``(name, image)``, a BGR uint8 (H, W, 3) array, built to reach one
corner of what ``cv2.imencode('.png', img)`` writes (see tests/png_encode_model.py)."""
from __future__ import annotations

import numpy as np

from tests import render_cases as rc


def from_filtered(rows):
    """The image whose Sub-filtered RGB scanlines are ``rows`` (h, 3 w): per channel a running sum along the row."""
    rows = np.asarray(rows, np.uint8)
    h, n = rows.shape
    rgb = np.cumsum(rows.reshape(h, n // 3, 3).astype(np.int64), axis=1) % 256
    return np.ascontiguousarray(rgb[:, :, ::-1].astype(np.uint8))


def distinct_stream(n, rng, first=1):
    """n random bytes, each different from the one before (``first`` precedes them): no run, so one literal each."""
    out = np.empty(n, np.uint8)
    prev = first
    for i, v in enumerate(rng.integers(1, 256, n)):
        prev = out[i] = (prev + v) % 256
    return out


def run_row(L):
    """One row whose scanline is the filter byte, then exactly L zero bytes, then a non-zero byte."""
    w = L // 3 + 1
    img = np.zeros((1, w, 3), np.uint8)
    img[0, -1, 2 - L % 3] = 9                # RGB channel L % 3 of the last pixel, the first one non-zero
    return img


def symbol_row(w, run, rng):
    """One row of w pixels whose 1 + 3 w scanline bytes are all literals but one run of ``run`` equal bytes, so the
    row has 1 + 3 w - run + 2 symbols (the run is a literal and one match)."""
    s = distinct_stream(3 * w, rng)
    at = len(s) // 2
    v = (int(s[at - 1]) + 128) % 256
    s[at:at + run] = v
    if s[at + run] == v:
        s[at + run] = (v + 1) % 256
    if s[at + run] == s[at + run + 1]:
        s[at + run] = (v + 2) % 256
    return from_filtered(s[None])


def fibonacci_row(rng):
    """Literal frequencies 1, 1, 2, 3, 5, ... over 18 byte values, no two equal bytes adjacent: a skewed histogram
    (gen_bitlen's repair past 15 bits is reached by the ``mixed`` cases)."""
    counts = [1, 1]
    while len(counts) < 18:
        counts.append(counts[-1] + counts[-2])
    vals = list(range(2, 2 + len(counts)))
    pool = {v: c for v, c in zip(vals, counts)}
    out, prev = [], 1
    while pool:
        v = max((u for u in pool if u != prev), key=lambda u: (pool[u], rng.random()), default=None)
        if v is None:
            break
        out.append(v)
        pool[v] -= 1
        if not pool[v]:
            del pool[v]
        prev = v
    while len(out) % 3:
        out.append(200 + len(out) % 3)
    return from_filtered(np.array(out, np.uint8)[None])


def mixed(h, w, seed):
    """Rows of noise, constant spans and a few values, at random lengths: runs of every length over block
    boundaries, literal / match mixes that make dynamic and static blocks."""
    rng = np.random.default_rng(seed)
    img = np.zeros((h, w, 3), np.uint8)
    for y in range(h):
        x = 0
        while x < w:
            n = int(rng.integers(1, max(2, w // 3)))
            kind = rng.integers(0, 3)
            if kind == 0:
                img[y, x:x + n] = rng.integers(0, 256, (min(n, w - x), 3))
            elif kind == 1:
                img[y, x:x + n] = rng.integers(0, 256, 3)
            else:
                img[y, x:x + n] = rng.integers(0, 3, (min(n, w - x), 3)) * 40
            x += n
    return img


def stored_multiple_of_8192():
    """Two rows of 4093 pixels whose 24 560 scanline bytes are all literals spread over all 256 values: two stored
    blocks (16383 bytes, then 8177), so the zlib stream is 2 + (1 + 4 + 16383) + (1 + 4 + 8177) + 4 = 24 576 =
    3 * 8192 bytes."""
    rng = np.random.default_rng(8192)
    s = distinct_stream(2 * (1 + 3 * 4093), rng)
    s = s.reshape(2, -1)
    s[:, 0] = 1
    for r in range(2):                       # the filter byte must not repeat its neighbours
        if s[r, 1] == 1:
            s[r, 1] = 2 if s[r, 2] != 2 else 3
        if r and s[r - 1, -1] == 1:
            s[r - 1, -1] = 4 if s[r - 1, -2] != 4 else 5
    return from_filtered(s[:, 1:])


def few_values(seed):
    """A small image of a few values; seed 184 makes a block whose dynamic and static sizes round to the same byte
    count (found by a seeded search), where zlib takes static."""
    rng = np.random.default_rng(seed)
    h, w = int(rng.integers(1, 12)), int(rng.integers(2, 40))
    k = int(rng.integers(2, 9))
    return (rng.integers(0, k, (h, w, 3)) * int(rng.integers(1, 60))).astype(np.uint8)


def cases():
    rng = np.random.default_rng(2024)
    out = []
    noise = lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    # width 1 (filter None) and height 1
    for h, w in ((1, 1), (5, 1), (300, 1), (1, 2), (1, 50), (1, 5000)):
        out.append(("noise_%dx%d" % (h, w), noise(h, w)))
        out.append(("const_%dx%d" % (h, w), np.full((h, w, 3), 7, np.uint8)))
    # every header window value: 4-20, 310, 4840, 12 660, 16 279 and >= 30 100 filtered bytes; 16 384 / 16 385
    for h, w in ((10, 10), (40, 40), (60, 70), (1, 5426), (100, 100), (1, 5461), (5, 1092)):
        out.append(("noise_%dx%d" % (h, w), noise(h, w)))
        out.append(("mixed_%dx%d" % (h, w), mixed(h, w, h * w)))
    # runs of 258..262 zero bytes (remainder 0..4), and longer ones
    for L in (3, 4, 5, 257, 258, 259, 260, 261, 262, 515, 516, 517, 774, 100000):
        out.append(("run_%d" % L, run_row(L)))
    out.append(("runs_stacked", np.concatenate([np.pad(run_row(L), ((0, 0), (0, 400 - run_row(L).shape[1]), (0, 0)))
                                                for L in range(255, 266)] * 6)))
    # 16383 and 32766 symbols: the final block is empty; 16384: it holds one symbol
    out.append(("sym_16383", symbol_row(5462, 6, rng)))
    out.append(("sym_32766", symbol_row(10925, 12, rng)))
    out.append(("sym_16384", symbol_row(5462, 5, rng)))
    out.append(("zstream_24576", stored_multiple_of_8192()))
    out.append(("fibonacci", fibonacci_row(rng)))
    out += [("tie_%d" % seed, few_values(seed)) for seed in (184, 366, 516)]
    out.append(("noise_300x400", noise(300, 400)))
    out.append(("zeros_480x640", np.zeros((480, 640, 3), np.uint8)))
    out.append(("three_values_37x1001", rng.integers(0, 3, (37, 1001, 3), dtype=np.uint8)))
    for k, (h, w) in enumerate(((97, 131), (200, 300), (256, 512), (333, 77))):
        out.append(("mixed_%dx%d" % (h, w), mixed(h, w, k)))
    out.append(("smooth_480x640", rc.image(480, 640, 5)))
    return out
