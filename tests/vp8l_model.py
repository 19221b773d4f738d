"""A plain-Python model of the lossless WebP (VP8L) decoder of RFC 9649, with libwebp's refusals, for the tests.

``decode(payload)`` takes the data from the VP8L payload (its signature byte) to the end of the file and returns the
decoded image as an (h, w) uint32 ARGB array, or raises ``Refused`` where libwebp (and so ``cv2.imread``) refuses the
stream.  ``groups(payload)`` reads as far as the main image's prefix-code groups and returns their count.  It is slow
(a Python loop per symbol) and meant for small files and for checking the device decoder's rules on CPU.
"""
from __future__ import annotations

import numpy as np

# RFC 9649 3.7.2.1.1: the order in which the code-length code's lengths are written
CODE_LENGTH_ORDER = (17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
# RFC 9649 4.2.2: (xi, yi) of distance codes 1..120; the distance is xi + yi * width, at least 1
DISTANCE_MAP = (
    (0, 1), (1, 0), (1, 1), (-1, 1), (0, 2), (2, 0), (1, 2), (-1, 2), (2, 1), (-2, 1), (2, 2), (-2, 2), (0, 3), (3, 0),
    (1, 3), (-1, 3), (3, 1), (-3, 1), (2, 3), (-2, 3), (3, 2), (-3, 2), (0, 4), (4, 0), (1, 4), (-1, 4), (4, 1),
    (-4, 1), (3, 3), (-3, 3), (2, 4), (-2, 4), (4, 2), (-4, 2), (0, 5), (3, 4), (-3, 4), (4, 3), (-4, 3), (5, 0),
    (1, 5), (-1, 5), (5, 1), (-5, 1), (2, 5), (-2, 5), (5, 2), (-5, 2), (4, 4), (-4, 4), (3, 5), (-3, 5), (5, 3),
    (-5, 3), (0, 6), (6, 0), (1, 6), (-1, 6), (6, 1), (-6, 1), (2, 6), (-2, 6), (6, 2), (-6, 2), (4, 5), (-4, 5),
    (5, 4), (-5, 4), (3, 6), (-3, 6), (6, 3), (-6, 3), (0, 7), (7, 0), (1, 7), (-1, 7), (5, 5), (-5, 5), (7, 1),
    (-7, 1), (4, 6), (-4, 6), (6, 4), (-6, 4), (2, 7), (-2, 7), (7, 2), (-7, 2), (3, 7), (-3, 7), (7, 3), (-7, 3),
    (5, 6), (-5, 6), (6, 5), (-6, 5), (8, 0), (4, 7), (-4, 7), (7, 4), (-7, 4), (8, 1), (8, 2), (6, 6), (-6, 6),
    (8, 3), (5, 7), (-5, 7), (7, 5), (-7, 5), (8, 4), (6, 7), (-6, 7), (7, 6), (-7, 6), (8, 5), (7, 7), (-7, 7),
    (8, 6), (8, 7))
assert len(DISTANCE_MAP) == 120
# alphabet sizes of the five codes of a group: green + length prefixes (+ cache), red, blue, alpha, distance
ALPHABET = (256 + 24, 256, 256, 256, 40)
PREDICTOR, CROSS_COLOR, SUBTRACT_GREEN, COLOR_INDEXING = range(4)


class Refused(ValueError):
    """libwebp refuses the stream."""


class Bits:
    """LSB-first reader.  Reading past the end yields zero bits; ``eos`` says more bits were read than exist, counting
    at least 8 bytes (libwebp loads 8 bytes up front), which libwebp refuses at the end of every header and image."""

    def __init__(self, data):
        self.d = bytes(data) + b"\0" * 8
        self.n = 8 * max(len(data), 8)
        self.p = 0

    def get(self, k):
        v = int.from_bytes(self.d[self.p >> 3:(self.p >> 3) + 5], "little") >> (self.p & 7) if self.p < self.n else 0
        self.p += k
        return v & ((1 << k) - 1)

    def peek(self, k):
        return int.from_bytes(self.d[self.p >> 3:(self.p >> 3) + 5], "little") >> (self.p & 7) & ((1 << k) - 1) \
            if self.p < self.n else 0

    @property
    def eos(self):
        return self.p > self.n


class Code:
    """A canonical prefix code from code lengths, refused as libwebp refuses it: all lengths zero, over-subscribed or
    incomplete, except a code with a single used symbol, which takes no bits."""

    def __init__(self, lengths):
        used = [s for s, l in enumerate(lengths) if l]
        if not used:
            raise Refused("no symbols")
        if len(used) == 1:
            self.single, self.bits = used[0], 0
            return
        self.single = None
        count = [0] * 16
        for l in lengths:
            count[l] += 1
        if sum(count[l] << (15 - l) for l in range(1, 16)) != 1 << 15:
            raise Refused("incomplete or over-subscribed code")
        self.bits = max(lengths)
        count[0] = 0
        nxt, code = [0] * 16, 0
        for l in range(1, 16):
            code = (code + count[l - 1]) << 1
            nxt[l] = code
        self.table = [None] * (1 << self.bits)
        for s, l in enumerate(lengths):
            if l:
                c = nxt[l]
                nxt[l] += 1
                rev = int(format(c, "0%db" % l)[::-1], 2)
                self.table[rev::1 << l] = [(s, l)] * len(range(rev, 1 << self.bits, 1 << l))

    def read(self, br):
        if self.single is not None:
            return self.single
        s, l = self.table[br.peek(self.bits)]
        br.p += l
        return s


def read_code(br, alphabet):
    """One prefix code (RFC 9649 3.7.2.1): simple (one or two symbols of up to 8 bits) or normal (code lengths coded
    with the code-length code, repeat codes 16/17/18, an optional max_symbol)."""
    lengths = [0] * alphabet
    if br.get(1):
        n = br.get(1) + 1
        s = br.get(8 if br.get(1) else 1)
        if s < alphabet:
            lengths[s] = 1
        if n == 2:
            s = br.get(8)
            if s < alphabet:
                lengths[s] = 1
    else:
        cl = [0] * 19
        for k in range(br.get(4) + 4):
            cl[CODE_LENGTH_ORDER[k]] = br.get(3)
        clc = Code(cl)
        if br.get(1):
            max_symbol = 2 + br.get(2 + 2 * br.get(3))
            if max_symbol > alphabet:
                raise Refused("max_symbol past the alphabet")
        else:
            max_symbol = alphabet
        s, prev = 0, 8
        while s < alphabet:
            if max_symbol == 0:
                break
            max_symbol -= 1
            c = clc.read(br)
            if c < 16:
                lengths[s] = c
                s += 1
                if c:
                    prev = c
            else:
                rep = br.get((2, 3, 7)[c - 16]) + (3, 3, 11)[c - 16]
                if s + rep > alphabet:
                    raise Refused("repeat past the alphabet")
                lengths[s:s + rep] = [prev if c == 16 else 0] * rep
                s += rep
    if br.eos:
        raise Refused("end of data")
    return Code(lengths)


def read_groups(br, count, cache_bits):
    return [[read_code(br, ALPHABET[j] + (1 << cache_bits if j == 0 and cache_bits else 0)) for j in range(5)]
            for _ in range(count)]


def prefix_value(sym, br):
    if sym < 4:
        return sym + 1
    extra = (sym - 2) >> 1
    return ((2 + (sym & 1)) << extra) + br.get(extra) + 1


def sub(size, bits):
    return (size + (1 << bits) - 1) >> bits


def decode_image(br, w, h, level0, stats=None):
    """The entropy-coded image of RFC 9649 5: w x h ARGB values (the main image at its coded width, or a sub-image)."""
    cache_bits = 0
    if br.get(1):
        cache_bits = br.get(4)
        if not 1 <= cache_bits <= 11:
            raise Refused("colour cache bits %d" % cache_bits)
    meta_bits, meta, ngroups = 0, None, 1
    if level0 and br.get(1):
        meta_bits = br.get(3) + 2
        mw = sub(w, meta_bits)
        meta = ((decode_image(br, mw, sub(h, meta_bits), False) >> 8) & 0xFFFF).reshape(-1)
        ngroups = int(meta.max()) + 1
    if br.eos:
        raise Refused("end of data")
    if stats is not None:
        stats["groups"] = ngroups
        return None
    groups = read_groups(br, ngroups, cache_bits)
    cache = [0] * (1 << cache_bits)
    out = np.zeros(w * h, np.uint32)
    pos, n = 0, w * h

    def push(v):
        if cache_bits:
            cache[((0x1E35A7BD * v) & 0xFFFFFFFF) >> (32 - cache_bits)] = v
        out[pos] = v

    while pos < n:
        y, x = divmod(pos, w)
        g = groups[int(meta[(y >> meta_bits) * mw + (x >> meta_bits)])] if meta is not None else groups[0]
        s = g[0].read(br)
        if s < 256:
            r, b, a = g[1].read(br), g[2].read(br), g[3].read(br)
            if br.eos:
                break
            push(a << 24 | r << 16 | s << 8 | b)
            pos += 1
        elif s < 256 + 24:
            length = prefix_value(s - 256, br)
            code = prefix_value(g[4].read(br), br)
            if code > 120:
                dist = code - 120
            else:
                xi, yi = DISTANCE_MAP[code - 1]
                dist = max(xi + yi * w, 1)
            if br.eos:
                break
            if dist > pos or length > n - pos:
                raise Refused("backward reference outside the image")
            for _ in range(length):
                push(int(out[pos - dist]))
                pos += 1
        else:
            if br.eos:
                break
            push(cache[s - 280])
            pos += 1
    if br.eos:
        raise Refused("end of data")
    return out.reshape(h, w)


def _avg(a, b):
    return (((a ^ b) & 0xFEFEFEFE) >> 1) + (a & b)


def _bytes(v):
    return [(v >> s) & 255 for s in (24, 16, 8, 0)]


def _pack(c):
    return c[0] << 24 | c[1] << 16 | c[2] << 8 | c[3]


def predict(mode, L, T, TL, TR):
    """libwebp's predictor of one pixel; modes 14 and 15 predict ARGB black as mode 0 does."""
    if mode in (0, 14, 15):
        return 0xFF000000
    if mode == 1:
        return L
    if mode == 2:
        return T
    if mode == 3:
        return TR
    if mode == 4:
        return TL
    if mode == 5:
        return _avg(_avg(L, TR), T)
    if mode == 6:
        return _avg(L, TL)
    if mode == 7:
        return _avg(L, T)
    if mode == 8:
        return _avg(TL, T)
    if mode == 9:
        return _avg(T, TR)
    if mode == 10:
        return _avg(_avg(L, TL), _avg(T, TR))
    if mode == 11:
        d = sum(abs(l - tl) - abs(t - tl) for l, t, tl in zip(_bytes(L), _bytes(T), _bytes(TL)))
        return T if d <= 0 else L
    if mode == 12:
        return _pack([min(max(l + t - tl, 0), 255) for l, t, tl in zip(_bytes(L), _bytes(T), _bytes(TL))])
    a = _bytes(_avg(L, T))
    return _pack([min(max(x + int((x - tl) / 2), 0), 255) for x, tl in zip(a, _bytes(TL))])


def _add(a, b):
    return (((a & 0xFF00FF00) + (b & 0xFF00FF00)) & 0xFF00FF00) | (((a & 0x00FF00FF) + (b & 0x00FF00FF)) & 0x00FF00FF)


def _s8(v):
    v &= 255
    return v - 256 if v > 127 else v


def inverse(t, img):
    """Undo one transform ``t = (type, bits, data, xsize)`` on the (h, xsize) image (its output width for colour
    indexing)."""
    kind, bits, data, xs = t
    h = img.shape[0]
    if kind == SUBTRACT_GREEN:
        g = (img >> 8) & 255
        return (img & 0xFF00FF00) | ((((img >> 16) + g) & 255) << 16) | ((img + g) & 255)
    if kind == COLOR_INDEXING:
        per = 8 >> bits
        x = np.arange(xs)
        idx = (img[:, x >> bits] >> 8 & 255) >> ((x & ((1 << bits) - 1)) * per) & ((1 << per) - 1)
        return data[idx]
    tw = sub(xs, bits)
    out = img.copy()
    if kind == CROSS_COLOR:
        for y in range(h):
            for x in range(xs):
                m = int(data[(y >> bits) * tw + (x >> bits)])
                v = int(img[y, x])
                g = _s8(v >> 8)
                r = ((v >> 16) + ((_s8(m) * g) >> 5)) & 255
                b = (v + ((_s8(m >> 8) * g) >> 5) + ((_s8(m >> 16) * _s8(r)) >> 5)) & 255
                out[y, x] = (v & 0xFF00FF00) | r << 16 | b
        return out
    flat = out.reshape(-1)
    for y in range(h):
        for x in range(xs):
            if y == 0:
                p = 0xFF000000 if x == 0 else int(flat[x - 1])
            elif x == 0:
                p = int(flat[(y - 1) * xs])
            else:
                i = y * xs + x
                mode = (int(data[(y >> bits) * tw + (x >> bits)]) >> 8) & 15
                # the top-right of the last column is the first pixel of the current row, as in a row-major buffer
                p = predict(mode, int(flat[i - 1]), int(flat[i - xs]), int(flat[i - xs - 1]), int(flat[i - xs + 1]))
            flat[y * xs + x] = _add(p, int(flat[y * xs + x]))
    return out


def read_header(payload):
    """(w, h) from the 5-byte VP8L header; raises ``Refused`` for a bad signature or version."""
    if len(payload) < 5 or payload[0] != 0x2F or payload[4] >> 5:
        raise Refused("bad VP8L header")
    v = int.from_bytes(payload[1:5], "little")
    return (v & 0x3FFF) + 1, ((v >> 14) & 0x3FFF) + 1


def read_transforms(br, w, h):
    """The transform list after the header: [(type, bits, data, xsize)] in reading order, and the coded width."""
    transforms, seen, xs = [], set(), w
    while br.get(1):
        kind = br.get(2)
        if kind in seen:
            raise Refused("transform %d twice" % kind)
        seen.add(kind)
        if kind in (PREDICTOR, CROSS_COLOR):
            bits = br.get(3) + 2
            data = decode_image(br, sub(xs, bits), sub(h, bits), False).reshape(-1)
            transforms.append((kind, bits, data, xs))
        elif kind == COLOR_INDEXING:
            n = br.get(8) + 1
            bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
            pal = decode_image(br, n, 1, False).reshape(-1)
            full = np.zeros(1 << (8 >> bits) if bits else 256, np.uint32)
            acc = 0
            for k in range(n):
                acc = _add(acc, int(pal[k]))
                full[k] = acc
            transforms.append((kind, bits, full, xs))
            xs = sub(xs, bits)
        else:
            transforms.append((kind, 0, None, xs))
    return transforms, xs


def transforms(payload):
    """The transforms of a stream, as ``read_transforms`` returns them."""
    w, h = read_header(payload)
    br = Bits(payload)
    br.p = 40
    return read_transforms(br, w, h)[0]


def decode(payload, stats=None):
    w, h = read_header(payload)
    br = Bits(payload)
    br.p = 40
    transforms, xs = read_transforms(br, w, h)
    img = decode_image(br, xs, h, True, stats)
    if stats is not None:
        return stats["groups"]
    for t in reversed(transforms):
        img = inverse(t, img)
    return img


def groups(payload):
    """The number of prefix-code groups the main image reads (the largest meta index plus one)."""
    return decode(payload, {})


def to_bgr(argb):
    return np.stack([argb & 255, (argb >> 8) & 255, (argb >> 16) & 255], -1).astype(np.uint8)
