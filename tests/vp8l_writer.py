"""A test-only lossless WebP (VP8L) writer that chooses the syntax elements itself: the transforms (with every
predictor mode, any cross-colour multipliers, palettes of any size with indices past the palette), the colour cache
size, simple or normal prefix codes with every repeat code and max_symbol, backward references (self-overlapping ones
too, through the distance map and past it) and an entropy image with group indices of its choosing, used or not.
cv2's encoder only exposes quality and method and never writes many of these.

``encode(argb, ...)`` returns ``(file, expected)``: the file's bytes and the ARGB image a decoder must produce
(equal to ``argb`` except where palette indices lie past the palette, which decode to 0).  ``matrix()`` is the seeded
set of files the tests run.
"""
from __future__ import annotations

import struct

import numpy as np

from tests.vp8l_model import (COLOR_INDEXING, CODE_LENGTH_ORDER, CROSS_COLOR, DISTANCE_MAP, PREDICTOR,
                              SUBTRACT_GREEN, _s8, predict, sub)


class BitWriter:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, v, k):
        self.v |= (v & ((1 << k) - 1)) << self.n
        self.n += k

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def balanced_lengths(counts, limit=15):
    """Complete code lengths for the used symbols: with k of them, the least frequent get ceil(log2 k) bits and the
    rest one bit less.  A single used symbol gets length 1 (a code of no bits)."""
    used = sorted((s for s, c in enumerate(counts) if c), key=lambda s: -counts[s])
    lengths = [0] * len(counts)
    if len(used) == 1:
        lengths[used[0]] = 1
        return lengths
    L = max(1, (len(used) - 1).bit_length())
    short = (1 << L) - len(used)                       # symbols at L - 1 bits
    assert L <= limit
    for i, s in enumerate(used):
        lengths[s] = L - 1 if i < short else L
    return lengths


def canonical(lengths):
    count = [0] * 16
    for l in lengths:
        if l:
            count[l] += 1
    nxt, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    codes = {}
    for s, l in enumerate(lengths):
        if l:
            codes[s] = (nxt[l], l)
            nxt[l] += 1
    return codes


def put_symbol(bw, codes, s):
    if len(codes) == 1:
        return                                         # a single-symbol code takes no bits
    c, l = codes[s]
    for k in range(l - 1, -1, -1):
        bw.put((c >> k) & 1, 1)


def _tokens(lengths, last):
    """Code-length symbols for lengths[:last]: literals 0..15, 16 (repeat the last non-zero length, 8 before any),
    17 and 18 (runs of zeros), with their extra bits."""
    tokens, i, prev = [], 0, 8
    while i < last:
        v = lengths[i]
        run = 1
        while i + run < last and lengths[i + run] == v:
            run += 1
        if v == 0 and run >= 3:
            r = min(run, 138)
            tokens.append((18, r - 11, 7) if r >= 11 else (17, r - 3, 3))
            i += r
        elif v and v == prev and run >= 3:
            r = min(run, 6)
            tokens.append((16, r - 3, 2))
            i += r
        else:
            tokens.append((v, 0, 0))
            if v:
                prev = v
            i += 1
    return tokens


def write_code(bw, counts, opt):
    """One prefix code for the symbol histogram ``counts``; returns its codes.  A simple code where the used symbols
    allow it and ``opt['simple']`` is set, else a normal code."""
    used = [s for s, c in enumerate(counts) if c] or [0]
    if opt.get("simple", True) and len(used) <= 2 and max(used) < 256:
        bw.put(1, 1)
        bw.put(len(used) - 1, 1)
        first = used[0]
        bw.put(first >= 2 or opt.get("wide", False), 1)
        bw.put(first, 8 if first >= 2 or opt.get("wide", False) else 1)
        if len(used) == 2:
            bw.put(used[1] if first == used[0] else used[0], 8)
        lengths = [0] * len(counts)
        for s in used:
            lengths[s] = 1
        return canonical(lengths)
    hist = list(counts)
    if not any(hist):
        hist[0] = 1
    lengths = balanced_lengths(hist)
    use_ms = opt.get("max_symbol", False)
    tokens = _tokens(lengths, max(s for s, l in enumerate(lengths) if l) + 1 if use_ms else len(lengths))
    if use_ms and len(tokens) < 2:                     # max_symbol counts at least two code-length symbols
        use_ms, tokens = False, _tokens(lengths, len(lengths))
    ch = [0] * 19
    for t, _, _ in tokens:
        ch[t] += 1
    cl = balanced_lengths(ch, 7)
    ncl = max([k + 1 for k in range(19) if cl[CODE_LENGTH_ORDER[k]]] + [4])
    bw.put(0, 1)
    bw.put(ncl - 4, 4)
    for k in range(ncl):
        bw.put(cl[CODE_LENGTH_ORDER[k]], 3)
    if opt.get("max_symbol_over"):                     # one past the alphabet: refused before any length is read
        use_ms, tokens = True, tokens[:2]
    if use_ms:
        ms = len(counts) + 1 if opt.get("max_symbol_over") else len(tokens)
        k = 0
        while ms - 2 >= 1 << (2 + 2 * k):
            k += 1
        bw.put(1, 1)
        bw.put(k, 3)
        bw.put(ms - 2, 2 + 2 * k)
    else:
        bw.put(0, 1)
    clc = canonical(cl)
    for t, extra, nb in tokens:
        put_symbol(bw, clc, t)
        bw.put(extra, nb)
    return canonical(lengths)


def prefix(v):
    """(symbol, extra bits, count) of a length or distance value >= 1."""
    if v <= 4:
        return v - 1, 0, 0
    x = v - 1
    h = x.bit_length() - 1
    second = (x >> (h - 1)) & 1
    return 2 * h + second, x & ((1 << (h - 1)) - 1), h - 1


def _plane_code(dist, w, use_map):
    if use_map:
        for k, (xi, yi) in enumerate(DISTANCE_MAP):
            if max(xi + yi * w, 1) == dist:
                return k + 1
    return dist + 120


def write_image(bw, px, w, h, opt, level0=False):
    """The entropy-coded image of the flat ARGB list ``px`` (w x h).  ``opt``: ``cache`` bits, ``copies`` (backward
    references for repeats, from the distances ``copy_dists``, default 1 and w), ``distance_map`` (False: code every
    distance past the map), ``code_opts`` (``simple``, ``wide``, ``max_symbol``, ``max_symbol_over``) and, at level 0,
    ``groups`` (k -> group index of 4 x 4 tile k; every group up to the largest is coded, used or not).  Streams
    libwebp refuses: ``cache_field`` writes that value as the colour cache bits (then codes without a cache),
    ``bad_copy`` = (pos, length, dist) codes that backward reference at pixel pos and ends the image there."""
    cache_bits = opt.get("cache", 0)
    if "cache_field" in opt:
        bw.put(1, 1)
        bw.put(opt["cache_field"], 4)
    elif cache_bits:
        bw.put(1, 1)
        bw.put(cache_bits, 4)
    else:
        bw.put(0, 1)
    tiles = None
    if level0:
        gmap = opt.get("groups")
        if gmap is None:
            bw.put(0, 1)
        else:
            bw.put(1, 1)
            bw.put(0, 3)                               # 4 x 4 tiles
            tw, th = sub(w, 2), sub(h, 2)
            tiles = [gmap(k) for k in range(tw * th)]
            write_image(bw, [g << 8 for g in tiles], tw, th, {})
    ngroups = max(tiles) + 1 if tiles else 1
    # the symbols, per group
    syms, cache, n, pos = [], [0] * (1 << cache_bits), len(px), 0
    use_map = opt.get("distance_map", True)

    def insert(v):
        if cache_bits:
            cache[((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - cache_bits)] = v

    while pos < n:
        y, x = divmod(pos, w)
        g = tiles[(y >> 2) * sub(w, 2) + (x >> 2)] if tiles else 0
        if opt.get("bad_copy") and pos == opt["bad_copy"][0]:
            syms.append((g, "copy", opt["bad_copy"][1], opt["bad_copy"][2]))
            break
        v = px[pos]
        run = 0
        if opt.get("copies") and pos:
            for dist in opt.get("copy_dists", lambda pos: (1, w))(pos):
                if 0 < dist <= pos:
                    r = 0
                    while pos + r < n and px[pos + r] == px[pos + r - dist] and r < 4096:
                        r += 1
                    if r >= 3:
                        run = r
                        break
        if run:
            syms.append((g, "copy", run, dist))
            for k in range(run):
                insert(px[pos + k])
            pos += run
            continue
        if cache_bits and cache[((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - cache_bits)] == v and pos % 3:
            syms.append((g, "cache", ((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - cache_bits)))
        else:
            syms.append((g, "lit", v))
        insert(v)
        pos += 1
    alpha = 280 + ((1 << cache_bits) if cache_bits else 0)
    hist = [[[0] * alpha, [0] * 256, [0] * 256, [0] * 256, [0] * 40] for _ in range(ngroups)]
    for s in syms:
        gh = hist[s[0]]
        if s[1] == "lit":
            v = s[2]
            gh[0][(v >> 8) & 255] += 1
            gh[1][(v >> 16) & 255] += 1
            gh[2][v & 255] += 1
            gh[3][v >> 24] += 1
        elif s[1] == "cache":
            gh[0][280 + s[2]] += 1
        else:
            gh[0][256 + prefix(s[2])[0]] += 1
            gh[4][prefix(_plane_code(s[3], w, use_map))[0]] += 1
    codes = [[write_code(bw, hist[g][j], opt.get("code_opts", {})) for j in range(5)] for g in range(ngroups)]
    for s in syms:
        c = codes[s[0]]
        if s[1] == "lit":
            v = s[2]
            put_symbol(bw, c[0], (v >> 8) & 255)
            put_symbol(bw, c[1], (v >> 16) & 255)
            put_symbol(bw, c[2], v & 255)
            put_symbol(bw, c[3], v >> 24)
        elif s[1] == "cache":
            put_symbol(bw, c[0], 280 + s[2])
        else:
            sym, extra, nb = prefix(s[2])
            put_symbol(bw, c[0], 256 + sym)
            bw.put(extra, nb)
            sym, extra, nb = prefix(_plane_code(s[3], w, use_map))
            put_symbol(bw, c[4], sym)
            bw.put(extra, nb)


def _fwd_predict(img, bits, modes):
    h, w = img.shape
    flat = [int(v) for v in img.reshape(-1)]
    out = list(flat)
    tw = sub(w, bits)
    for y in range(h):
        for x in range(w):
            i = y * w + x
            if y == 0:
                p = 0xFF000000 if x == 0 else flat[i - 1]
            elif x == 0:
                p = flat[i - w]
            else:
                p = predict(modes[(y >> bits) * tw + (x >> bits)], flat[i - 1], flat[i - w], flat[i - w - 1],
                            flat[i - w + 1])
            out[i] = _sub(flat[i], p)
    return np.array(out, np.uint32).reshape(h, w)


def _sub(a, b):
    return (((a | 0x00FF00FF) - (b & 0xFF00FF00)) & 0xFF00FF00) | (((a | 0xFF00FF00) - (b & 0x00FF00FF)) & 0x00FF00FF)


def encode(argb, transforms=(), opt=None, palette=None, indices=None):
    """A simple-container VP8L file.  ``transforms``: a list of (type, params) applied in order; PREDICTOR takes
    (bits, modes per tile), CROSS_COLOR (bits, (g2r, g2b, r2b) per tile), SUBTRACT_GREEN None, COLOR_INDEXING
    needs ``palette`` (n ARGB values) and ``indices`` (h x w), and must come first."""
    opt = opt or {}
    if indices is not None:
        h, w = indices.shape
        full = np.zeros(256, np.uint32)
        full[:len(palette)] = palette
        argb = full[indices]
    h, w = argb.shape
    expected = argb.copy()
    bw = BitWriter()
    bw.put(0x2F, 8)
    bw.put(w - 1, 14)
    bw.put(h - 1, 14)
    bw.put(0, 1)                                       # alpha hint
    bw.put(0, 3)
    img = argb
    for kind, params in transforms:
        bw.put(1, 1)
        bw.put(kind, 2)
        if kind == SUBTRACT_GREEN:
            g = (img >> 8) & 255
            img = (img & 0xFF00FF00) | ((((img >> 16) - g) & 255) << 16) | ((img - g) & 255)
        elif kind == PREDICTOR:
            bits, modes = params
            bw.put(bits - 2, 3)
            tw, th = sub(img.shape[1], bits), sub(h, bits)
            write_image(bw, [m << 8 for m in modes[:tw * th]], tw, th, {})
            img = _fwd_predict(img, bits, modes)
        elif kind == CROSS_COLOR:
            bits, mults = params
            bw.put(bits - 2, 3)
            tw, th = sub(img.shape[1], bits), sub(h, bits)
            m = [((c[2] & 255) << 16) | ((c[1] & 255) << 8) | (c[0] & 255) for c in mults[:tw * th]]
            write_image(bw, m, tw, th, {})
            out = img.copy()
            for y in range(h):
                for x in range(img.shape[1]):
                    g2r, g2b, r2b = mults[(y >> bits) * tw + (x >> bits)]
                    v = int(img[y, x])
                    gg, rr = _s8(v >> 8), (v >> 16) & 255
                    r = (rr - ((g2r * gg) >> 5)) & 255
                    b = ((v & 255) - ((g2b * gg) >> 5) - ((r2b * _s8(rr)) >> 5)) & 255
                    out[y, x] = (v & 0xFF00FF00) | r << 16 | b
            img = out
        else:
            n = len(palette)
            bw.put(n - 1, 8)
            bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
            deltas = [int(palette[0])] + [_sub(int(palette[k]), int(palette[k - 1])) for k in range(1, n)]
            write_image(bw, deltas, n, 1, opt.get("palette_opt", {}))
            per = 8 >> bits
            pw = sub(w, bits)
            packed = np.zeros((h, pw), np.uint32)
            for x in range(w):
                packed[:, x >> bits] |= (indices[:, x].astype(np.uint32) << ((x & ((1 << bits) - 1)) * per))
            img = packed << 8 | 0xFF000000
    bw.put(0, 1)
    write_image(bw, [int(v) for v in img.reshape(-1)], img.shape[1], h, opt, level0=True)
    payload = bw.bytes()
    ch = b"VP8L" + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) & 1 else b"")
    return b"RIFF" + struct.pack("<I", 4 + len(ch)) + b"WEBP" + ch, expected


def _argb(h, w, seed, levels=256, alpha=False):
    rng = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 7 + y * 3 + k * 40) % 256 for k in range(3)], -1)
    noise = rng.randint(0, 256, (h, w, 3))
    c = np.where(rng.rand(h, w, 1) < 0.3, noise, base) // (256 // levels) * (256 // levels)
    a = rng.randint(0, 256, (h, w)) if alpha else np.full((h, w), 255)
    return (a.astype(np.uint32) << 24 | c[..., 2].astype(np.uint32) << 16 | c[..., 1].astype(np.uint32) << 8
            | c[..., 0].astype(np.uint32))


def matrix():
    """[(name, file, expected ARGB)] over the branches: simple 1- and 2-symbol codes (1- and 8-bit first symbols),
    normal codes with max_symbol and every repeat code, all 16 predictor modes at tile sizes 4 to 16, cross-colour
    with negative multipliers, 2/4/16/256-colour palettes with indices past the palette, cache sizes 1 to 11,
    self-overlapping copies through the distance map and past it, unused group indices, and one file over the group
    budget (65 groups).  ``copy_bounds`` holds a copy whose distance is every pixel decoded so far and whose length
    reaches the last pixel, the largest ones libwebp accepts."""
    out = []

    def add(name, *a, **k):
        f, e = encode(*a, **k)
        out.append((name, f, e))

    flat = np.full((5, 7), 0xFF102030, np.uint32)
    add("flat_simple1", flat)                                        # every code a single symbol: no bits
    two = np.where(np.arange(35).reshape(5, 7) % 3, 0xFF010001, 0xFF000100).astype(np.uint32)
    add("two_simple2", two)
    add("two_simple_wide", two, opt={"code_opts": {"wide": True}})
    add("two_normal", two, opt={"code_opts": {"simple": False}})
    for k, (h, w) in enumerate([(1, 1), (1, 17), (9, 1), (13, 21), (33, 40)]):
        im = _argb(h, w, k, alpha=k % 2 == 1)
        add("normal_ms_%dx%d" % (h, w), im, opt={"code_opts": {"simple": False, "max_symbol": True}})
        add("copies_%dx%d" % (h, w), np.repeat(im[:, :max(1, w // 3)], 3, 1)[:, :w] if w > 2 else im,
            opt={"copies": True, "code_opts": {"simple": False}})
    smooth = _argb(20, 23, 5, levels=4)
    add("copies_past_map", smooth, opt={"copies": True, "distance_map": False})
    period = np.array([0xFF000000 | (k * 0x10305) for k in range(7)], np.uint32)
    add("copy_bounds", np.tile(period, 5).reshape(5, 7), opt={"copies": True, "copy_dists": lambda pos: (pos,)})
    for bits in range(1, 12):
        add("cache_%d" % bits, _argb(17, 19, 10 + bits, levels=8), opt={"cache": bits, "copies": bits % 2 == 0})
    # every predictor mode, tiles of 4, 8 and 16
    for bits in (2, 3, 4):
        h, w = 37, 41
        tw, th = sub(w, bits), sub(h, bits)
        modes = [(k * 5 + bits) % 16 for k in range(tw * th)]
        if bits == 2:
            modes = [k % 16 for k in range(tw * th)]
        add("predictor_%d" % bits, _argb(h, w, 20 + bits, alpha=True), [(PREDICTOR, (bits, modes))])
    # negative and positive cross-colour multipliers, after subtract-green and a predictor
    rng = np.random.RandomState(3)
    h, w = 29, 35
    mults = [tuple(int(v) for v in rng.randint(-128, 128, 3)) for _ in range(sub(w, 2) * sub(h, 2))]
    mults[0] = (-128, -1, 127)
    add("cross_color", _argb(h, w, 30), [(CROSS_COLOR, (2, mults))])
    modes = [11, 12, 13, 14, 15, 5, 10, 3] * 40
    add("all_transforms", _argb(h, w, 31, alpha=True),
        [(SUBTRACT_GREEN, None), (PREDICTOR, (2, modes)), (CROSS_COLOR, (3, mults))], {"cache": 4, "copies": True})
    # palettes: 2 / 4 / 16 / 256 colours, and sizes that leave index room past the palette
    for n, extra in ((2, 0), (3, 1), (4, 0), (11, 5), (16, 0), (200, 56), (256, 0)):
        pal = np.array(_argb(1, n, 40 + n, alpha=True)[0], np.uint32)
        h, w = 11, 37
        top = n + extra
        idx = np.random.RandomState(n).randint(0, top, (h, w)).astype(np.uint8)
        add("palette_%d_%d" % (n, extra), None, [(COLOR_INDEXING, None)], palette=pal, indices=idx)
    pal = np.array([0xFF0000FF, 0xFF00FF00, 0x80FF0000], np.uint32)
    idx = np.random.RandomState(9).randint(0, 4, (19, 23)).astype(np.uint8)
    add("palette_predictor", None, [(COLOR_INDEXING, None), (PREDICTOR, (2, list(range(16)) * 4))], palette=pal,
        indices=idx)
    # entropy images: groups 0 and 3 used, 1 and 2 coded but unused; 64 groups (the budget) and 65 (over it)
    add("groups_unused", _argb(24, 24, 50), opt={"groups": lambda k: 3 * (k % 2)})
    big = _argb(40, 40, 51)
    add("groups_64", big, opt={"groups": lambda k: k % 64})
    add("groups_65", big, opt={"groups": lambda k: k % 65})
    return out


def refused():
    """[(name, file, reason)]: streams libwebp refuses past the header, each at one check, with the refusal
    ``tests.vp8l_model`` names: a backward reference further back than the pixels decoded so far, one whose length
    runs past the last pixel, a transform read twice, colour cache bits of 0 and of 12 and 15, a max_symbol past the
    alphabet."""
    im = _argb(6, 7, 60)
    n = im.size
    cases = [("distance_before_start", im, (), {"bad_copy": (5, 2, 6)}, "backward reference"),
             ("distance_before_start_row", im, (), {"bad_copy": (6, 1, 7)}, "backward reference"),
             ("copy_past_end", im, (), {"bad_copy": (n - 2, 3, 1)}, "backward reference"),
             ("copy_past_end_long", im, (), {"bad_copy": (1, n, 1)}, "backward reference"),
             ("transform_twice", im, [(SUBTRACT_GREEN, None), (SUBTRACT_GREEN, None)], {}, "transform 2 twice"),
             ("predictor_twice", im, [(PREDICTOR, (2, [1] * 4)), (PREDICTOR, (2, [1] * 4))], {}, "transform 0 twice"),
             ("cache_bits_0", im, (), {"cache_field": 0}, "colour cache bits 0"),
             ("cache_bits_12", im, (), {"cache_field": 12}, "colour cache bits 12"),
             ("cache_bits_15", im, (), {"cache_field": 15}, "colour cache bits 15"),
             ("max_symbol_past_alphabet", im, (), {"code_opts": {"simple": False, "max_symbol_over": True}},
              "max_symbol past the alphabet")]
    return [(name, encode(a, t, o)[0], reason) for name, a, t, o, reason in cases]
