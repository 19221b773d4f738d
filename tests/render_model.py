"""Plain-Python model of the cv2 rasterisation the pose renderer reproduces (``csrc/render.cu``), for the tests.

cv2 does not document which pixels its drawing calls touch.  These functions state them, and ``test_render_cpu.py``
pins each one equal to cv2 on seeded random shapes:
  * ``line_pixels``: ``cv2.line(..., 1, LINE_8)`` between integer points, clipped to the image first;
  * ``convex_mask``: ``cv2.fillConvexPoly(..., LINE_8, shift=0)``, the edges' lines plus one span per row;
  * ``convex_rows``: the same pixels as one [lo, hi] interval per row, the form the kernel stores;
  * ``rect_mask``: ``cv2.rectangle(..., thickness=2)``, three-pixel bands with plus-shaped corner caps;
  * ``circle2_mask``: ``cv2.circle(..., 2, thickness=-1)``, a 13-pixel diamond.
All integer arithmetic is C's: 64-bit, arithmetic right shift, division truncated toward zero.
"""
from __future__ import annotations

import numpy as np

XY_SHIFT = 16


def _cdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def clip_line(w, h, x1, y1, x2, y2):
    """cv2's ``clipLine`` on the (w, h) image: ``(visible, x1, y1, x2, y2)``, with the same truncation."""
    right, bottom = w - 1, h - 1
    if w <= 0 or h <= 0:
        return False, x1, y1, x2, y2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def line_pixels(w, h, x1, y1, x2, y2):
    """The (x, y) pixels of an 8-connected line, walked left to right after clipping."""
    if not (0 <= x1 < w and 0 <= x2 < w and 0 <= y1 < h and 0 <= y2 < h):
        ok, x1, y1, x2, y2 = clip_line(w, h, x1, y1, x2, y2)
        if not ok:
            return []
    dx, dy = x2 - x1, y2 - y1
    sx = sy = 1
    if dx < 0:
        dx, dy = -dx, -dy
        x1, y1, x2, y2 = x2, y2, x1, y1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
        sx, sy = sy, sx
    err, plus, minus = dx - (dy + dy), dx + dx, -(dy + dy)
    # x/y step taken every pixel (minus) and on an error carry (plus)
    mx, my, px, py = sx, 0, 0, sy
    if vert:
        mx, my, px, py = my, mx, py, px
    x, y, out = x1, y1, []
    for _ in range(dx + 1):
        out.append((x, y))
        carry = err < 0
        err += minus + (plus if carry else 0)
        x += mx + (px if carry else 0)
        y += my + (py if carry else 0)
    return out


def convex_spans(w, h, pts):
    """The scanline part of ``fillConvexPoly`` (shift 0, LINE_8): ``[(y, x_lo, x_hi)]`` clipped to the image, and
    whether the polygon is drawn at all (cv2 returns before any span when it lies wholly outside)."""
    n = len(pts)
    xs = [int(p[0]) for p in pts]
    ys = [int(p[1]) for p in pts]
    imin = int(np.argmin(ys))
    ymin, ymax, xmin, xmax = ys[imin], max(ys), min(xs), max(xs)
    if n < 3 or xmax < 0 or ymax < 0 or xmin >= w or ymin >= h:
        return []
    ymax = min(ymax, h - 1)
    half = 1 << (XY_SHIFT - 1)
    edges = n
    e = [dict(idx=imin, di=1, x=-(1 << XY_SHIFT), dx=0, ye=ymin), dict(idx=imin, di=n - 1, x=-(1 << XY_SHIFT), dx=0, ye=ymin)]
    y, out = ymin, []
    while True:
        for ed in e:
            if y >= ed["ye"]:
                idx0 = ed["idx"]
                idx = (idx0 + ed["di"]) % n
                while edges > 0:
                    edges -= 1
                    ty = ys[idx]
                    if ty > y:
                        xs0, xe0 = xs[idx0] << XY_SHIFT, xs[idx] << XY_SHIFT
                        ed["ye"] = ty
                        ed["dx"] = _cdiv((xe0 - xs0) * 2 + (ty - y), 2 * (ty - y))
                        ed["x"] = xs0
                        ed["idx"] = idx
                        break
                    idx0 = idx
                    idx = (idx + ed["di"]) % n
                else:
                    edges -= 1
        if edges < 0:
            break
        if y >= 0:
            l, r = (1, 0) if e[0]["x"] > e[1]["x"] else (0, 1)
            x1 = (e[l]["x"] + half) >> XY_SHIFT
            x2 = (e[r]["x"] + half) >> XY_SHIFT
            if x2 >= 0 and x1 < w:
                x1, x2 = max(x1, 0), min(x2, w - 1)
                if x1 <= x2:
                    out.append((y, x1, x2))
        e[0]["x"] += e[0]["dx"]
        e[1]["x"] += e[1]["dx"]
        y += 1
        if y > ymax:
            break
    return out


def convex_mask(w, h, pts):
    """``fillConvexPoly(img, pts, c, LINE_8, 0)``'s pixels: every edge's line, then the spans."""
    m = np.zeros((h, w), bool)
    n = len(pts)
    for i in range(n):
        (xa, ya), (xb, yb) = pts[i - 1], pts[i]
        for x, y in line_pixels(w, h, int(xa), int(ya), int(xb), int(yb)):
            m[y, x] = True
    for y, a, b in convex_spans(w, h, pts):
        m[y, a:b + 1] = True
    return m


def convex_rows(w, h, pts):
    """``convex_mask`` as ``{y: (lo, hi)}``: each row's leftmost and rightmost pixel."""
    rows = {}
    n = len(pts)

    def add(y, a, b):
        lo, hi = rows.get(y, (a, b))
        rows[y] = (min(lo, a), max(hi, b))
    for i in range(n):
        (xa, ya), (xb, yb) = pts[i - 1], pts[i]
        for x, y in line_pixels(w, h, int(xa), int(ya), int(xb), int(yb)):
            add(y, x, x)
    for y, a, b in convex_spans(w, h, pts):
        add(y, a, b)
    return rows


def _fill(m, xa, ya, xb, yb):
    h, w = m.shape
    xa, xb, ya, yb = max(xa, 0), min(xb, w - 1), max(ya, 0), min(yb, h - 1)
    if xa <= xb and ya <= yb:
        m[ya:yb + 1, xa:xb + 1] = True


def rect_mask(w, h, x1, y1, x2, y2):
    """``cv2.rectangle(img, (x1, y1), (x2, y2), c, 2)``: each non-degenerate side is a three-pixel band between its
    corners, and each corner gets a plus of radius 1 (cv2's round cap of a two-pixel line)."""
    m = np.zeros((h, w), bool)
    lx, hx, ly, hy = min(x1, x2), max(x1, x2), min(y1, y2), max(y1, y2)
    if x1 != x2:
        _fill(m, lx, y1 - 1, hx, y1 + 1)
        _fill(m, lx, y2 - 1, hx, y2 + 1)
    if y1 != y2:
        _fill(m, x1 - 1, ly, x1 + 1, hy)
        _fill(m, x2 - 1, ly, x2 + 1, hy)
    for cx, cy in ((x1, y1), (x2, y1), (x1, y2), (x2, y2)):
        _fill(m, cx - 1, cy, cx + 1, cy)
        _fill(m, cx, cy - 1, cx, cy + 1)
    return m


def circle2_mask(w, h, x, y):
    """``cv2.circle(img, (x, y), 2, c, -1)``: rows y-2..y+2 with half-widths 0, 1, 2, 1, 0."""
    m = np.zeros((h, w), bool)
    for dy, r in ((-2, 0), (-1, 1), (0, 2), (1, 1), (2, 0)):
        _fill(m, x - r, y + dy, x + r, y + dy)
    return m
