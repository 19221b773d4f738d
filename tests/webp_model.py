"""A numpy model of the device WebP decoder's stages after the entropy decode (csrc/webp.cu), run on the syntax
elements a ``tests.webp_writer.Frame`` wrote: dequantisation and the inverse WHT, intra prediction and the inverse
DCT in raster order, libwebp's loop filter in raster order, then fancy upsampling and libwebp's YUV -> BGR.  It is
written from RFC 6386 and libwebp's documented behaviour, independently of the kernels' wavefront order, so the CPU
tests can hold it against cv2.imdecode."""
from __future__ import annotations

import numpy as np

from tests.webp_writer import B_DC, B_HD, B_HE, B_HU, B_LD, B_RD, B_TM, B_VE, B_VL, B_VR, ZIGZAG


def _clip8(v):
    return min(max(int(v), 0), 255)


def _wrap16(v):
    return ((int(v) + 32768) & 0xFFFF) - 32768


def _iwht(c):
    t = [0] * 16
    for i in range(4):
        a0, a1 = c[i] + c[12 + i], c[4 + i] + c[8 + i]
        a2, a3 = c[4 + i] - c[8 + i], c[i] - c[12 + i]
        t[i], t[8 + i], t[4 + i], t[12 + i] = a0 + a1, a0 - a1, a3 + a2, a3 - a2
    out = [0] * 16
    for i in range(4):
        dc = t[4 * i] + 3
        a0, a1 = dc + t[4 * i + 3], t[4 * i + 1] + t[4 * i + 2]
        a2, a3 = t[4 * i + 1] - t[4 * i + 2], dc - t[4 * i + 3]
        out[4 * i:4 * i + 4] = [(a0 + a1) >> 3, (a3 + a2) >> 3, (a0 - a1) >> 3, (a3 - a2) >> 3]
    return out


def _idct_add(c, blk):
    """The inverse DCT of raster coefficients ``c`` added to the 4x4 array ``blk`` in place."""
    m1 = lambda a: ((a * 20091) >> 16) + a
    m2 = lambda a: (a * 35468) >> 16
    t = [0] * 16
    for i in range(4):
        a, b = c[i] + c[8 + i], c[i] - c[8 + i]
        cc, d = m2(c[4 + i]) - m1(c[12 + i]), m1(c[4 + i]) + m2(c[12 + i])
        t[4 * i:4 * i + 4] = [a + d, b + cc, b - cc, a - d]
    for i in range(4):
        dc = t[i] + 4
        a, b = dc + t[8 + i], dc - t[8 + i]
        cc, d = m2(t[4 + i]) - m1(t[12 + i]), m1(t[4 + i]) + m2(t[12 + i])
        for x, v in enumerate((a + d, b + cc, b - cc, a - d)):
            blk[i, x] = _clip8(int(blk[i, x]) + (v >> 3))


def _avg3(a, b, c):
    return (a + 2 * b + c + 2) >> 2


def _avg2(a, b):
    return (a + b + 1) >> 1


def _pred4(top, left, tl, mode):
    """4x4 prediction from the 8 pixels above (4 above-right), the 4 to the left and the corner."""
    A, B, C, D, E, F, G, H = top
    I, J, K, L = left
    X = tl
    p = np.zeros((4, 4), np.int64)
    if mode == B_DC:
        p[:] = (sum(top[:4]) + sum(left) + 4) >> 3
    elif mode == B_TM:
        for y in range(4):
            for x in range(4):
                p[y, x] = _clip8(top[x] + left[y] - X)
    elif mode == B_VE:
        p[:] = [_avg3(X, A, B), _avg3(A, B, C), _avg3(B, C, D), _avg3(C, D, E)]
    elif mode == B_HE:
        p[:] = np.array([_avg3(X, I, J), _avg3(I, J, K), _avg3(J, K, L), _avg3(K, L, L)])[:, None]
    else:
        # diagonal modes as position -> value tables, (x, y)
        if mode == B_RD:
            e = [L, K, J, I, X, A, B, C, D]                          # the edge from bottom-left to top-right
            for y in range(4):
                for x in range(4):
                    k = 3 - y + x + 1                                   # index of the centre sample on the edge
                    p[y, x] = _avg3(e[k - 1], e[k], e[k + 1])
        elif mode == B_LD:
            e = [A, B, C, D, E, F, G, H, H]
            for y in range(4):
                for x in range(4):
                    k = x + y
                    p[y, x] = _avg3(e[k], e[k + 1], e[k + 2])
        elif mode == B_VR:
            t = {(0, 0): _avg2(X, A), (1, 0): _avg2(A, B), (2, 0): _avg2(B, C), (3, 0): _avg2(C, D),
                 (0, 3): _avg3(K, J, I), (0, 2): _avg3(J, I, X), (0, 1): _avg3(I, X, A), (1, 1): _avg3(X, A, B),
                 (2, 1): _avg3(A, B, C), (3, 1): _avg3(B, C, D)}
            t.update({(1, 2): t[0, 0], (2, 2): t[1, 0], (3, 2): t[2, 0], (1, 3): t[0, 1], (2, 3): t[1, 1],
                      (3, 3): t[2, 1]})
            for (x, y), v in t.items():
                p[y, x] = v
        elif mode == B_VL:
            t = {(0, 0): _avg2(A, B), (1, 0): _avg2(B, C), (2, 0): _avg2(C, D), (3, 0): _avg2(D, E),
                 (0, 1): _avg3(A, B, C), (1, 1): _avg3(B, C, D), (2, 1): _avg3(C, D, E), (3, 1): _avg3(D, E, F),
                 (3, 2): _avg3(E, F, G), (3, 3): _avg3(F, G, H)}
            t.update({(0, 2): t[1, 0], (1, 2): t[2, 0], (2, 2): t[3, 0], (0, 3): t[1, 1], (1, 3): t[2, 1],
                      (2, 3): t[3, 1]})
            for (x, y), v in t.items():
                p[y, x] = v
        elif mode == B_HD:
            t = {(0, 0): _avg2(I, X), (0, 1): _avg2(J, I), (0, 2): _avg2(K, J), (0, 3): _avg2(L, K),
                 (3, 0): _avg3(A, B, C), (2, 0): _avg3(X, A, B), (1, 0): _avg3(I, X, A), (1, 1): _avg3(J, I, X),
                 (1, 2): _avg3(K, J, I), (1, 3): _avg3(L, K, J)}
            t.update({(2, 1): t[0, 0], (2, 2): t[0, 1], (2, 3): t[0, 2], (3, 1): t[1, 0], (3, 2): t[1, 1],
                      (3, 3): t[1, 2]})
            for (x, y), v in t.items():
                p[y, x] = v
        else:
            assert mode == B_HU
            t = {(0, 0): _avg2(I, J), (2, 0): _avg2(J, K), (2, 1): _avg2(K, L), (1, 0): _avg3(I, J, K),
                 (3, 0): _avg3(J, K, L), (3, 1): _avg3(K, L, L)}
            t.update({(0, 1): t[2, 0], (0, 2): t[2, 1], (1, 1): t[3, 0], (1, 2): t[3, 1]})
            for (x, y), v in t.items():
                p[y, x] = v
            for x, y in ((3, 2), (2, 2), (0, 3), (1, 3), (2, 3), (3, 3)):
                p[y, x] = L
    return p


def _pred_block(top, left, tl, n, mode, mb_x, mb_y):
    """n x n luma or chroma prediction; DC at the frame's edges averages what exists, 128 at the corner."""
    p = np.zeros((n, n), np.int64)
    sh = 4 if n == 16 else 3
    if mode == B_DC:
        if mb_x and mb_y:
            p[:] = (sum(top) + sum(left) + n) >> (sh + 1)
        elif mb_y:
            p[:] = (sum(top) + n // 2) >> sh
        elif mb_x:
            p[:] = (sum(left) + n // 2) >> sh
        else:
            p[:] = 128
    elif mode == B_TM:
        for y in range(n):
            for x in range(n):
                p[y, x] = _clip8(top[x] + left[y] - tl)
    elif mode == B_VE:
        p[:] = np.array(top)[None, :]
    else:
        p[:] = np.array(left)[:, None]
    return p


def _planes(frame):
    """Reconstructed (unfiltered) Y, U, V planes padded to whole macroblocks, plus each macroblock's
    (i4x4, has non-zero coefficients) for the loop filter."""
    mbw, mbh = (frame.w + 15) >> 4, (frame.h + 15) >> 4
    Y = np.zeros((16 * mbh, 16 * mbw), np.int64)
    U = np.zeros((8 * mbh, 8 * mbw), np.int64)
    V = np.zeros_like(U)
    nonzero = []
    use_skip = frame.skip_prob is not None
    for my in range(mbh):
        for mx in range(mbw):
            mb = frame.mbs[my * mbw + mx]
            y1dc, y1ac, y2dc, y2ac, uvdc, uvac = frame.steps(mb.segment)
            lv = np.zeros((25, 16), np.int64) if use_skip and mb.skip else mb.levels
            coef = np.zeros((24, 16), np.int64)                 # raster order per block
            for b in range(24):
                dc, ac = (uvdc, uvac) if b >= 16 else (y1dc, y1ac)
                for n in range(16):
                    coef[b, ZIGZAG[n]] = _wrap16(int(lv[b, n]) * (dc if n == 0 else ac))
            if not mb.i4x4:
                y2 = [0] * 16
                for n in range(16):
                    y2[ZIGZAG[n]] = _wrap16(int(lv[24, n]) * (y2dc if n == 0 else y2ac))
                coef[:16, 0] = [_wrap16(v) for v in _iwht(y2)]
            # libwebp's "any non-zero coefficient": a level past the first position, or a non-zero DC, in a block
            nonzero.append(bool(((lv[:24, 1:] != 0).any(axis=1) | (coef[:, 0] != 0)).any()))
            x0, y0 = 16 * mx, 16 * my
            # the 16 + 4 pixels above (127 above the frame; above-right from the row above, replicated at the right
            # edge), the 16 to the left (129 left of the frame), the corner (127 on the first row, else 129 at x = 0)
            if my:
                top = list(Y[y0 - 1, x0:x0 + 16])
                top += list(Y[y0 - 1, x0 + 16:x0 + 20]) if mx < mbw - 1 else [Y[y0 - 1, x0 + 15]] * 4
                tl = Y[y0 - 1, x0 - 1] if mx else 129
            else:
                top, tl = [127] * 20, 127
            left = list(Y[y0:y0 + 16, x0 - 1]) if mx else [129] * 16
            if mb.i4x4:
                for n in range(16):
                    sy, sx = n >> 2, n & 3
                    by, bx = y0 + 4 * sy, x0 + 4 * sx
                    if sy == 0:
                        t8 = top[4 * sx:4 * sx + 8]
                    else:
                        t8 = list(Y[by - 1, bx:bx + 4]) + (list(Y[by - 1, bx + 4:bx + 8]) if sx < 3 else top[16:20])
                    l4 = list(Y[by:by + 4, bx - 1]) if sx else left[4 * sy:4 * sy + 4]
                    if sx and sy:
                        c = Y[by - 1, bx - 1]
                    elif sy:
                        c = left[4 * sy - 1]
                    elif sx:
                        c = top[4 * sx - 1]
                    else:
                        c = tl
                    blk = _pred4([int(v) for v in t8], [int(v) for v in l4], int(c), mb.imodes[n])
                    _idct_add(list(coef[n]), blk)
                    Y[by:by + 4, bx:bx + 4] = blk
            else:
                blk = _pred_block([int(v) for v in top[:16]], [int(v) for v in left], int(tl), 16, mb.ymode, mx, my)
                for n in range(16):
                    sy, sx = n >> 2, n & 3
                    sub = blk[4 * sy:4 * sy + 4, 4 * sx:4 * sx + 4]
                    _idct_add(list(coef[n]), sub)
                Y[y0:y0 + 16, x0:x0 + 16] = blk
            for P, base in ((U, 16), (V, 20)):
                cx0, cy0 = 8 * mx, 8 * my
                if my:
                    ct = [int(v) for v in P[cy0 - 1, cx0:cx0 + 8]]
                    ctl = int(P[cy0 - 1, cx0 - 1]) if mx else 129
                else:
                    ct, ctl = [127] * 8, 127
                cl = [int(v) for v in P[cy0:cy0 + 8, cx0 - 1]] if mx else [129] * 8
                blk = _pred_block(ct, cl, ctl, 8, mb.uvmode, mx, my)
                for n in range(4):
                    sy, sx = n >> 1, n & 1
                    _idct_add(list(coef[base + n]), blk[4 * sy:4 * sy + 4, 4 * sx:4 * sx + 4])
                P[cy0:cy0 + 8, cx0:cx0 + 8] = blk
    return Y, U, V, nonzero


def _filter_params(frame, segment, i4x4):
    """(limit, interior limit, HEV threshold) as libwebp computes them; limit 0: not filtered."""
    if frame.level == 0:
        return 0, 0, 0
    level = frame.level
    if frame.use_segment:
        level = (frame.seg_filter[segment] or 0) if frame.update_data else 0
        if frame.update_data and not frame.absolute:
            level += frame.level
    if frame.use_lf_delta and frame.update_lf_delta:
        level += frame.ref_deltas[0] or 0
        if i4x4:
            level += frame.mode_deltas[0] or 0
    level = min(max(level, 0), 63)
    if level == 0:
        return 0, 0, 0
    il = level
    if frame.sharpness:
        il >>= 2 if frame.sharpness > 4 else 1
        il = min(il, 9 - frame.sharpness)
    il = max(il, 1)
    return 2 * level + il, il, 2 if level >= 40 else 1 if level >= 15 else 0


def _edge(P, pts, hev_t, t, it, kind):
    """Filter across one edge at the given pixel lines; ``pts`` are lists of 8 (row, col) from p3 to q3."""
    sc1 = lambda v: min(max(v, -128), 127)
    sc2 = lambda v: min(max(v, -16), 15)
    t2 = 2 * t + 1
    for line in pts:
        v = [int(P[r, c]) for r, c in line]
        p3, p2, p1, p0, q0, q1, q2, q3 = v
        if 4 * abs(p0 - q0) + abs(p1 - q1) > t2:
            continue
        if kind != "simple" and not all(abs(a - b) <= it for a, b in ((p3, p2), (p2, p1), (p1, p0), (q3, q2),
                                                                        (q2, q1), (q1, q0))):
            continue
        hev = kind != "simple" and (abs(p1 - p0) > hev_t or abs(q1 - q0) > hev_t)
        if kind == "simple" or hev:
            a = 3 * (q0 - p0) + sc1(p1 - q1)
            a1, a2 = sc2((a + 4) >> 3), sc2((a + 3) >> 3)
            out = {3: p0 + a2, 4: q0 - a1}
        elif kind == "edge":
            a = sc1(3 * (q0 - p0) + sc1(p1 - q1))
            a1, a2, a3 = (27 * a + 63) >> 7, (18 * a + 63) >> 7, (9 * a + 63) >> 7
            out = {1: p2 + a3, 2: p1 + a2, 3: p0 + a1, 4: q0 - a1, 5: q1 - a2, 6: q2 - a3}
        else:
            a = 3 * (q0 - p0)
            a1, a2 = sc2((a + 4) >> 3), sc2((a + 3) >> 3)
            a3 = (a1 + 1) >> 1
            out = {2: p1 + a3, 3: p0 + a2, 4: q0 - a1, 5: q1 - a3}
        for k, val in out.items():
            P[line[k]] = _clip8(val)


def _loop_filter(frame, Y, U, V, nonzero):
    mbw, mbh = (frame.w + 15) >> 4, (frame.h + 15) >> 4
    simple = frame.simple
    for my in range(mbh):
        for mx in range(mbw):
            mb = frame.mbs[my * mbw + mx]
            limit, il, hev_t = _filter_params(frame, mb.segment, mb.i4x4)
            if limit == 0:
                continue
            inner = mb.i4x4 or nonzero[my * mbw + mx]
            planes = [(Y, 16)] if simple else [(Y, 16), (U, 8), (V, 8)]
            for vertical in (True, False):          # vertical edges (left, inner), then horizontal (top, inner)
                for P, n in planes:
                    x0, y0 = n * mx, n * my
                    # edges at offset 0 (macroblock edge) and 4, 8, 12 (luma) or 4 (chroma)
                    offs = ([0] if (mx if vertical else my) else []) + ([4, 8, 12] if n == 16 else [4]) * inner
                    for o in offs:
                        if vertical:
                            pts = [[(y0 + j, x0 + o + k) for k in range(-4, 4)] for j in range(n)]
                        else:
                            pts = [[(y0 + o + k, x0 + j) for k in range(-4, 4)] for j in range(n)]
                        kind = "simple" if simple else "edge" if o == 0 else "inner"
                        _edge(P, pts, hev_t, limit + 4 if o == 0 else limit, il, kind)


def _bgr(Y, U, V, h, w):
    out = np.zeros((h, w, 3), np.uint8)

    def up(C, y, x):
        ny, nx = y >> 1, x >> 1
        fy = 0 if y == 0 else ny + 1 if y & 1 else ny - 1
        fy = ny if fy > (h - 1) >> 1 else fy
        fx = 0 if x == 0 else nx + 1 if x & 1 else nx - 1
        fx = nx if fx > (w - 1) >> 1 else fx
        nn, fn = int(C[ny, nx]), int(C[fy, nx])
        if fx == nx:
            return (3 * nn + fn + 2) >> 2
        nf, ff = int(C[ny, fx]), int(C[fy, fx])
        return (((nn + 3 * nf + 3 * fn + ff + 8) >> 3) + nn) >> 1

    clip = lambda v: v >> 6 if (v & ~16383) == 0 else 0 if v < 0 else 255
    for y in range(h):
        for x in range(w):
            yy = (int(Y[y, x]) * 19077) >> 8
            u, v = up(U, y, x), up(V, y, x)
            out[y, x] = (clip(yy + ((u * 33050) >> 8) - 17685),
                         clip(yy - ((u * 6419) >> 8) - ((v * 13320) >> 8) + 8708),
                         clip(yy + ((v * 26149) >> 8) - 14234))
    return out


def decode(frame):
    """What cv2.imread gives for ``frame.encode()``: the (h, w, 3) uint8 BGR image."""
    Y, U, V, nonzero = _planes(frame)
    _loop_filter(frame, Y, U, V, nonzero)
    return _bgr(Y, U, V, frame.h, frame.w)
