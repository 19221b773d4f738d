"""A test-only JPEG writer (T.81 Huffman coding) that takes quantised coefficient blocks as they are, with no rate or
quality search.  Every header and entropy-coding choice is a knob, so a decoder can be driven through files unlike
cv2.imencode's: 16-bit DQT, table ids 0-3, optimised / long-code / single-symbol / all-ones Huffman tables, arbitrary
component ids and sampling factors, tables after SOF, APPn / COM segments and fill bytes between markers, restart
intervals of any length, a missing EOI or bytes after it, and progressive scan scripts with DC successive approximation,
arbitrary AC bands, AC refinement with correction bits, long EOB runs and DHT / DRI changes between scans.

``Frame(...).encode()`` returns the file.  Coefficients are per component an int array (block rows, blocks per row, 64)
in natural (row-major) order, covering whole MCUs.  ``corpus()`` is the conformance corpus of the JPEG tests: named
files, each with the route the device decoder must give it (see ``Case``)."""
from __future__ import annotations

import functools
import struct
from dataclasses import dataclass, field

import numpy as np

from centerpose_b200.jpeg import IDCT_RANGE, ZIGZAG

# libjpeg's jpeg_simple_progression for three components and for one, (components, Ss, Se, Ah, Al)
SIMPLE_YCC = [([0, 1, 2], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([2], 1, 63, 0, 1), ([1], 1, 63, 0, 1), ([0], 6, 63, 0, 2),
              ([0], 1, 63, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([2], 1, 63, 1, 0), ([1], 1, 63, 1, 0), ([0], 1, 63, 1, 0)]
SIMPLE_GRAY = [([0], 0, 0, 0, 1), ([0], 1, 5, 0, 2), ([0], 6, 63, 0, 2), ([0], 1, 63, 2, 1), ([0], 0, 0, 1, 0),
               ([0], 1, 63, 1, 0)]


@functools.lru_cache(None)
def _annex_k():
    """The T.81 Annex K tables as libjpeg writes them: Huffman tables K.3 ((class, id) -> (bits, values)) and the
    quantisation tables K.1 (natural order, luminance and chrominance), read back from a file cv2 writes at quality 50
    with its default (standard) Huffman tables."""
    import cv2
    from centerpose_b200 import jpeg
    ok, buf = cv2.imencode(".jpg", np.zeros((8, 8, 3), np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 50])
    d = buf.tobytes()
    huff, qt, pos = {}, {}, 2
    while d[pos + 1] != 0xDA:
        m, ln = d[pos + 1], struct.unpack(">H", d[pos + 2:pos + 4])[0]
        seg = d[pos + 4:pos + 2 + ln]
        if m == 0xC4:
            jpeg._read_dht(seg, huff, "annex k")
        elif m == 0xDB:
            for o in range(0, len(seg), 65):
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = np.frombuffer(seg, np.uint8, 64, o + 1)
                qt[seg[o] & 15] = nat
        pos += 2 + ln
    return {k: (list(v[0]), list(v[1])) for k, v in huff.items()}, qt


def quant_table(quality, chroma=False):
    """libjpeg's jpeg_quality_scaling of the Annex K table, limited to 1..255."""
    base = _annex_k()[1][1 if chroma else 0]
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * scale + 50) // 100, 1, 255)


# ---- Huffman tables -------------------------------------------------------------------------------------------------

def optimal_table(freq):
    """T.81 K.2's code lengths for the symbol counts ``freq`` (symbol -> count), limited to 16 bits, one code point of
    the longest length kept free (so no code is all ones): (bits[16], values)."""
    f = np.zeros(257, np.int64)
    for s, c in freq.items():
        f[s] = c
    f[256] = 1
    size, others = [0] * 257, [-1] * 257
    while True:
        live = [i for i in range(257) if f[i]]
        if len(live) < 2:
            break
        c1 = min(live, key=lambda i: (f[i], -i))
        c2 = min((i for i in live if i != c1), key=lambda i: (f[i], -i))
        f[c1] += f[c2]
        f[c2] = 0
        for c in (c1, c2):
            size[c] += 1
            while others[c] >= 0:
                c = others[c]
                size[c] += 1
        c = c1
        while others[c] >= 0:
            c = others[c]
        others[c] = c2
    bits = [0] * 33
    for i in range(257):
        if size[i]:
            bits[size[i]] += 1
    for i in range(32, 16, -1):
        while bits[i]:
            j = i - 2
            while not bits[j]:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while not bits[i]:
        i -= 1
    bits[i] -= 1
    vals = [s for ln in range(1, 33) for s in range(256) if size[s] == ln]
    return bits[1:17], vals


def long_table(freq, dc):
    """A table with most codes longer than LUT_BITS = 9: the eight most frequent symbols get lengths 2..9, every other
    symbol (padded to all 12 DC categories, or to 64 AC symbols) lengths 10..16 in turn."""
    syms = sorted(freq, key=lambda s: (-freq[s], s))
    pool = range(12) if dc else range(256)
    syms += [s for s in pool if s not in freq][:max(0, (12 if dc else 64) - len(syms))]
    lengths = {s: 2 + i if i < 8 else 10 + (i - 8) % 7 for i, s in enumerate(syms)}
    assert sum(2.0 ** -ln for ln in lengths.values()) < 1
    bits = [sum(1 for v in lengths.values() if v == ln) for ln in range(1, 17)]
    return bits, sorted(syms, key=lambda s: (lengths[s], syms.index(s)))


def make_table(kind, freq, dc, all_ones=False):
    """(bits, values) of a table of ``kind`` ("annexk" for id 0 / 1 of ``dc``'s class, "optimal", "long", "single")
    covering the symbols of ``freq``.  ``all_ones`` adds one unused symbol at the longest length, whose code is then all
    ones (T.81 C forbids it; libjpeg refuses the table)."""
    if kind.startswith("annexk"):
        bits, vals = _annex_k()[0][(0 if dc else 1, int(kind[-1]) if kind[-1].isdigit() else 0)]
        assert set(freq) <= set(vals), "symbols outside the Annex K table"
    elif kind == "optimal":
        bits, vals = optimal_table(freq)
    elif kind == "long":
        bits, vals = long_table(freq, dc)
    elif kind == "single":
        assert len(freq) == 1, "a single-symbol table codes one symbol"
        bits, vals = [1] + [0] * 15, list(freq)
    else:
        raise ValueError(kind)
    bits, vals = list(bits), list(vals)
    if all_ones:
        ln = max(i for i in range(16) if bits[i]) + 1
        bits[ln - 1] += 1
        vals.append(next(s for s in range(16 if dc else 256) if s not in vals))
        assert codes(bits, vals)[vals[-1]] == ((1 << ln) - 1, ln), "the table has room for more than one code"
    return bits, vals


def codes(bits, vals):
    """symbol -> (code, length) of the canonical code (T.81 C.2)."""
    out, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            out[vals[k]] = (code, ln)
            code += 1
            k += 1
        code <<= 1
    return out


# ---- entropy coding as events: ("sym", table key, symbol), ("bits", value, n), ("rst",) ------------------------------

def _category(v):
    return int(abs(int(v))).bit_length()


def _value(v, s):
    """The s low bits that code v (T.81 F.1.2.1)."""
    return int(v) if v >= 0 else int(v) + (1 << s) - 1


def _eob(eobrun, key):
    n = eobrun.bit_length() - 1
    yield "sym", key, n << 4
    if n:
        yield "bits", eobrun - (1 << n), n


@dataclass
class Frame:
    """One JPEG file.  ``comps`` lists per component (id, h, v, quant table, DC table, AC table); ``coef`` the
    quantised blocks per component (whole MCUs), ``qt`` quant table id -> 64 values (natural order).  ``huff`` is a
    table kind for every table, or a dict ((class, id) -> kind); ``script`` a progressive scan list (component
    indices, Ss, Se, Ah, Al), None for one sequential scan."""
    h: int
    w: int
    comps: list
    coef: list
    qt: dict
    sof: int = 0xC0
    qt16: bool = False
    huff: object = "optimal"
    all_ones: tuple = None                  # (class, id) of a table to give an all-ones code
    ri: int = 0
    ri_per_scan: list = None                # progressive: the restart interval of each scan (a DRI before it)
    dht_per_scan: bool = False              # progressive: each scan's tables, in a DHT right before its SOS
    tables_after_sof: bool = False
    extras: bool = False                    # APPn and COM segments between the header markers and between scans
    fill: bool = False                      # fill bytes (0xFF) before every marker
    jfif: bool = True
    eoi: bool = True
    trailer: bytes = b""
    script: list = None
    _out: bytearray = field(default=None, repr=False)

    # ---- geometry ----
    @property
    def hmax(self):
        return max(c[1] for c in self.comps)

    @property
    def vmax(self):
        return max(c[2] for c in self.comps)

    def mcus(self):
        return -(-self.w // (8 * self.hmax)), -(-self.h // (8 * self.vmax))

    def coded_blocks(self, i):
        """(blocks per row, block rows) of component i alone (T.81 A.2.2)."""
        _, hs, vs = self.comps[i][:3]
        return -(-(-(-self.w * hs // self.hmax)) // 8), -(-(-(-self.h * vs // self.vmax)) // 8)

    def units(self, idx):
        """Per unit of a scan over components ``idx``: its blocks as (component, block row, block column)."""
        if len(idx) == 1:
            bw, bh = self.coded_blocks(idx[0])
            return [[(idx[0], by, bx)] for by in range(bh) for bx in range(bw)]
        mx, my = self.mcus()
        out = []
        for y in range(my):
            for x in range(mx):
                out.append([(i, y * self.comps[i][2] + dy, x * self.comps[i][1] + dx) for i in idx
                            for dy in range(self.comps[i][2]) for dx in range(self.comps[i][1])])
        return out

    # ---- entropy coding ----
    def _sequential(self, ri):
        idx = list(range(len(self.comps)))
        pred = [0] * len(idx)
        for u, blocks in enumerate(self.units(idx)):
            if ri and u and u % ri == 0:
                yield ("rst",)
                pred = [0] * len(idx)
            for i, by, bx in blocks:
                blk = self.coef[i][by, bx]
                d = int(blk[0]) - pred[i]
                pred[i] = int(blk[0])
                s = _category(d)
                yield "sym", (0, self.comps[i][4]), s
                yield "bits", _value(d, s), s
                r = 0
                for k in range(1, 64):
                    v = int(blk[ZIGZAG[k]])
                    if not v:
                        r += 1
                        continue
                    while r > 15:
                        yield "sym", (1, self.comps[i][5]), 0xF0
                        r -= 16
                    s = _category(v)
                    yield "sym", (1, self.comps[i][5]), (r << 4) | s
                    yield "bits", _value(v, s), s
                    r = 0
                if r:
                    yield "sym", (1, self.comps[i][5]), 0

    def _progressive(self, scan, ri):
        idx, ss, se, ah, al = scan
        units = self.units(idx)
        pred, eobrun, pending = [0] * len(self.comps), 0, []
        key = (1, self.comps[idx[0]][5])
        for u, blocks in enumerate(units):
            if ri and u and u % ri == 0:
                if eobrun:
                    yield from _eob(eobrun, key)
                    yield from (("bits", b, 1) for b in pending)
                    eobrun, pending = 0, []
                yield ("rst",)
                pred = [0] * len(self.comps)
            for i, by, bx in blocks:
                blk = [int(v) for v in self.coef[i][by, bx][ZIGZAG]]       # zigzag order
                if ss == 0 and not ah:
                    v = blk[0] >> al
                    d, pred[i] = v - pred[i], v
                    s = _category(d)
                    yield "sym", (0, self.comps[i][4]), s
                    yield "bits", _value(d, s), s
                elif ss == 0:
                    yield "bits", (blk[0] >> al) & 1, 1
                elif not ah:                                    # AC first (T.81 G.1.2.2)
                    r = 0
                    for k in range(ss, se + 1):
                        a = abs(blk[k]) >> al
                        if not a:
                            r += 1
                            continue
                        if eobrun:
                            yield from _eob(eobrun, key)
                            eobrun = 0
                        while r > 15:
                            yield "sym", key, 0xF0
                            r -= 16
                        s = _category(a)
                        yield "sym", key, (r << 4) | s
                        yield "bits", _value(a if blk[k] > 0 else -a, s), s
                        r = 0
                    if r:
                        eobrun += 1
                        if eobrun == 0x7FFF:
                            yield from _eob(eobrun, key)
                            eobrun = 0
                else:                                           # AC refinement (T.81 G.1.2.3)
                    a = [abs(blk[k]) >> al for k in range(64)]
                    last = max([k for k in range(ss, se + 1) if a[k] == 1], default=-1)
                    r, corr = 0, []
                    for k in range(ss, se + 1):
                        if not a[k]:
                            r += 1
                            continue
                        while r > 15 and k <= last:
                            if eobrun:
                                yield from _eob(eobrun, key)
                                yield from (("bits", b, 1) for b in pending)
                                eobrun, pending = 0, []
                            yield "sym", key, 0xF0
                            r -= 16
                            yield from (("bits", b, 1) for b in corr)
                            corr = []
                        if a[k] > 1:                            # nonzero history: a correction bit
                            corr.append(a[k] & 1)
                            continue
                        if eobrun:
                            yield from _eob(eobrun, key)
                            yield from (("bits", b, 1) for b in pending)
                            eobrun, pending = 0, []
                        yield "sym", key, (r << 4) | 1
                        yield "bits", int(blk[k] > 0), 1
                        yield from (("bits", b, 1) for b in corr)
                        corr, r = [], 0
                    if r or corr:
                        eobrun += 1
                        pending += corr
                        if eobrun == 0x7FFF:
                            yield from _eob(eobrun, key)
                            yield from (("bits", b, 1) for b in pending)
                            eobrun, pending = 0, []
        if eobrun:
            yield from _eob(eobrun, key)
            yield from (("bits", b, 1) for b in pending)

    # ---- bytes ----
    def _marker(self, m, payload=None):
        if self.fill:
            self._out += b"\xFF\xFF"
        self._out += bytes([0xFF, m])
        if payload is not None:
            self._out += struct.pack(">H", len(payload) + 2) + payload

    def _extras(self, n):
        if self.extras:
            self._marker(0xFE, b"comment %d" % n)
            self._marker(0xE5, b"APP5 payload")

    def _dht(self, tables):
        if tables:
            self._marker(0xC4, b"".join(bytes([c << 4 | t] + list(bits) + list(vals))
                                        for (c, t), (bits, vals) in sorted(tables.items())))

    def _tables(self, events):
        freq = {}
        for e in events:
            if e[0] == "sym":
                freq.setdefault(e[1], {}).setdefault(e[2], 0)
                freq[e[1]][e[2]] += 1
        kinds = self.huff if isinstance(self.huff, dict) else {k: self.huff for k in freq}
        return {k: make_table(kinds[k], f, k[0] == 0, self.all_ones == k) for k, f in freq.items()}

    def _scan_data(self, events, tables):
        cd = {k: codes(*t) for k, t in tables.items()}
        acc, n, out, rst = 0, 0, bytearray(), 0

        def flush():
            nonlocal acc, n
            while n >= 8:
                b = (acc >> (n - 8)) & 255
                out.append(b)
                if b == 0xFF:
                    out.append(0)
                n -= 8
            acc &= (1 << n) - 1

        for e in events:
            if e[0] == "sym":
                c, ln = cd[e[1]][e[2]]
                acc, n = (acc << ln) | c, n + ln
            elif e[0] == "bits":
                acc, n = (acc << e[2]) | e[1], n + e[2]
            else:
                if n % 8:
                    pad = 8 - n % 8
                    acc, n = (acc << pad) | ((1 << pad) - 1), n + pad
                flush()
                if self.fill:
                    out += b"\xFF"
                out += bytes([0xFF, 0xD0 + rst % 8])
                rst += 1
            flush()
        if n:
            pad = 8 - n
            acc, n = (acc << pad) | ((1 << pad) - 1), 8
            flush()
        return out

    def encode(self):
        self._out = bytearray(b"\xFF\xD8")
        if self.jfif:
            self._marker(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
        self._extras(0)
        progressive = self.script is not None
        scans = self.script if progressive else [None]
        ris = self.ri_per_scan or [self.ri] * len(scans)
        events = [list(self._progressive(s, r) if progressive else self._sequential(r)) for s, r in zip(scans, ris)]
        per_scan = [self._tables(e) for e in events] if self.dht_per_scan else None
        tables = self._tables([x for e in events for x in e]) if not per_scan else per_scan[0]
        qts = b"".join(bytes([(16 if self.qt16 else 0) | t]) +
                       (struct.pack(">64H", *(int(v) for v in np.asarray(q)[ZIGZAG])) if self.qt16
                        else bytes(int(v) for v in np.asarray(q)[ZIGZAG])) for t, q in sorted(self.qt.items()))
        sof = struct.pack(">BHHB", 8, self.h, self.w, len(self.comps)) + b"".join(
            bytes([cid, hs << 4 | vs, tq]) for cid, hs, vs, tq, _, _ in self.comps)
        if not self.tables_after_sof:
            self._marker(0xDB, qts)
            self._extras(1)
        else:
            self._marker(self.sof, sof)
            self._extras(1)
        self._dht(tables)
        self._extras(2)
        if ris[0] or self.ri_per_scan:
            self._marker(0xDD, struct.pack(">H", ris[0]))
        if self.tables_after_sof:
            self._marker(0xDB, qts)
        else:
            self._marker(self.sof, sof)
        self._extras(3)
        for n, (scan, ev) in enumerate(zip(scans, events)):
            if n:
                self._extras(10 + n)
                if per_scan:
                    self._dht(per_scan[n])
                if ris[n] != ris[n - 1]:
                    self._marker(0xDD, struct.pack(">H", ris[n]))
            idx, ss, se, ah, al = scan if progressive else (list(range(len(self.comps))), 0, 63, 0, 0)
            self._marker(0xDA, bytes([len(idx)]) + b"".join(
                bytes([self.comps[i][0], self.comps[i][4] << 4 | self.comps[i][5]]) for i in idx) +
                bytes([ss, se, ah << 4 | al]))
            self._out += self._scan_data(ev, per_scan[n] if per_scan else tables)
        if self.eoi:
            self._marker(0xD9)
        self._out += self.trailer
        return bytes(self._out)


# ---- coefficient sources --------------------------------------------------------------------------------------------

def _dct_matrix():
    k = np.arange(8)
    m = np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16) * np.sqrt(2 / 8)
    m[0] /= np.sqrt(2)
    return m


def fdct_blocks(plane, q):
    """The orthonormal 2-D DCT of every 8x8 block of an (8 bh, 8 bw) uint8 plane, level shifted, quantised by q
    (natural order) with rounding: (bh, bw, 64) -- the coefficients an encoder writes (libjpeg's scaling)."""
    bh, bw = plane.shape[0] // 8, plane.shape[1] // 8
    m = _dct_matrix()
    b = plane.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3).astype(np.float64) - 128
    f = np.einsum("ui,abij,vj->abuv", m, b, m).reshape(bh, bw, 64)
    return np.rint(f / np.asarray(q)).astype(np.int64)


def smooth_plane(rng, h, w, noise=10.0):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    ph = rng.uniform(0, 6, 2)
    im = 127.5 + 110 * np.sin(x / max(w, 2) * rng.uniform(1, 5) + y / max(h, 2) * rng.uniform(1, 4) + ph[0])
    return np.clip(np.rint(im + rng.normal(0, noise, im.shape)), 0, 255).astype(np.uint8)


def image_coefs(rng, comps, h, w, qt, noise=10.0):
    """Legitimate-regime blocks: the quantised forward DCT of a seeded image plane per component (whole MCUs)."""
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    return [fdct_blocks(smooth_plane(rng, my * c[2] * 8, mx * c[1] * 8, noise), qt[c[3]]) for c in comps]


def sparse_coefs(rng, comps, h, w, amp=40, density=0.1, dc=200):
    """Random sparse blocks: each AC coefficient nonzero with probability ``density``, uniform in +-amp."""
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    out = []
    for c in comps:
        shape = (my * c[2], mx * c[1], 64)
        b = rng.randint(-amp, amp + 1, shape) * (rng.uniform(size=shape) < density)
        b[..., 0] = rng.randint(-dc, dc + 1, shape[:2])
        out.append(b.astype(np.int64))
    return out


# ---- the IDCT range check, restated --------------------------------------------------------------------------------

def _pass1_matrix():
    """Pass 1 of libjpeg's ISLOW IDCT on one column as integer weights: out[n] = (sum_k M[n, k] x[k] + 2^10) >> 11."""
    from tests.test_jpeg_cpu import _idct_1d
    return _idct_1d(np.eye(8, dtype=np.int64) << 11, 11)


def pass1_peak(blocks, q):
    """The largest magnitude among the dequantised coefficients and pass-1 outputs of each block (..., 64)."""
    from tests.test_jpeg_cpu import _idct_1d
    x = np.asarray(blocks, np.int64) * np.asarray(q, np.int64)
    cols = x.reshape(-1, 8, 8).transpose(1, 2, 0)                   # (row u, column v, block)
    p1 = np.abs(_idct_1d(cols, 11)).max((0, 1)).reshape(x.shape[:-1])
    return np.maximum(np.abs(x).max(-1), p1)


def block_in_range(blocks, q):
    """Per block: whether every dequantised coefficient and every pass-1 output of the ISLOW IDCT lies within
    +-IDCT_RANGE (the device decodes those blocks and flags the rest)."""
    return pass1_peak(blocks, q) <= IDCT_RANGE


def boundary_block(rng, target, row=0):
    """A natural-order block (q = 1) whose largest pass-1 output is ``target``: every column carries the sign
    pattern of IDCT output ``row`` at a random share of the amplitude, the amplitude is bisected to the last value
    at or below ``target``, then single coefficients are stepped by one until the peak is ``target``."""
    m = _pass1_matrix()
    s = np.where(m[row] < 0, -1, 1)
    spread = np.r_[1.0, rng.uniform(0.3, 1.0, 7)]
    make = lambda a: np.rint(np.outer(s, spread) * a).astype(np.int64).reshape(64)
    peak = lambda b: int(pass1_peak(b, 1))
    lo, hi = 0.0, float(target)
    for _ in range(50):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if peak(make(mid)) <= target else (lo, mid)
    blk = make(lo)
    while peak(blk) < target:
        best = None
        for i in range(64):
            for d in (1, -1):
                b2 = blk.copy()
                b2[i] += d
                p = peak(b2)
                if peak(blk) < p <= target and (best is None or p > best[0]):
                    best = (p, b2)
        if best is None:
            break
        blk = best[1]
    return blk


# ---- the conformance corpus -----------------------------------------------------------------------------------------

@dataclass
class Case:
    """A corpus file and its route.  ``route``: "device" (the parser takes it, the device decodes it with status 0),
    "range" (the parser takes it, the device flags blocks outside the IDCT's 16-bit range: status 1), "corrupt" (the
    parser takes it, the entropy data is bad or ends early: status 1), "no_eoi" (the parser takes it with ``eoi``
    False, the device flags it without decoding: status 1), "host" (``parse`` says not eligible, ``why`` in its
    reason), "raise" (``parse`` raises, ``why`` in the message)."""
    name: str
    data: bytes
    route: str
    why: str = ""
    legit: bool = False                  # coefficients of a real image (the model must equal cv2 on them)


YCC = [(1, 2, 2, 0, 0, 0), (2, 1, 1, 1, 1, 1), (3, 1, 1, 1, 1, 1)]


def _ycc(luma=(2, 2), ids=(1, 2, 3), tq=(0, 1, 1), td=(0, 1, 1), ta=(0, 1, 1), chroma=(1, 1)):
    return [(ids[0], luma[0], luma[1], tq[0], td[0], ta[0]), (ids[1], chroma[0], chroma[1], tq[1], td[1], ta[1]),
            (ids[2], 1, 1, tq[2], td[2], ta[2])]


def _frame(rng, comps, h, w, quality=75, source="image", **kw):
    qt = {c[3]: quant_table(quality, c[3] % 2 == 1) for c in comps}
    coef = (image_coefs(rng, comps, h, w, qt) if source == "image"
            else sparse_coefs(rng, comps, h, w))
    return Frame(h, w, comps, coef, qt, **kw)


def corrupt_entropy(data):
    """The file with 128 one-bits (stuffed 0xFF bytes) spliced into its first scan's entropy data: more than a code
    and its value bits can take, and no code of a table that keeps the all-ones code point free matches the rest."""
    sos = data.index(b"\xFF\xDA")
    at = sos + 2 + struct.unpack(">H", data[sos + 2:sos + 4])[0] + 3
    return data[:at] + b"\xFF\x00" * 16 + data[at:]


@functools.lru_cache(None)
def corpus():
    """The conformance corpus: a few hundred seeded files over every knob, each with its route."""
    rng = np.random.RandomState(20261018)
    out = []

    def add(name, frame_or_data, route="device", why="", legit=None):
        data = frame_or_data.encode() if isinstance(frame_or_data, Frame) else frame_or_data
        out.append(Case(name, data, route, why, legit if legit is not None else route == "device"))

    sizes = [(1, 1), (7, 13), (16, 16), (23, 41), (40, 56), (61, 37)]
    lumas = [(1, 1), (2, 1), (1, 2), (2, 2)]
    kinds = ["annexk", "optimal", "long"]
    # sequential: samplings x sizes x table kinds, restart intervals 1 / not dividing the MCU row / beyond the image
    for li, luma in enumerate(lumas):
        for si, (h, w) in enumerate(sizes):
            kind = kinds[(li + si) % 3]
            huff = {(0, 0): "annexk0", (1, 0): "annexk0", (0, 1): "annexk1", (1, 1): "annexk1"} \
                if kind == "annexk" else kind
            ri = [0, 1, 3, 1000][(li * 7 + si) % 4]
            q = [50, 75, 95, 100][(li + 2 * si) % 4]
            add("seq_%dx%d_%dx%d_%s_ri%d" % (luma + (h, w) + (kind, ri)),
                _frame(rng, _ycc(luma), h, w, q, huff=huff, ri=ri, sof=0xC0 if si % 2 else 0xC1))
    # grayscale, declared (1, 1) and (2, 2)
    for n, (h, w) in enumerate(sizes):
        comps = [(7 + n, 2 if n % 2 else 1, 2 if n % 2 else 1, n % 4, n % 4, (n + 1) % 4)]
        add("gray_%dx%d_decl%d" % (h, w, comps[0][1]),
            _frame(rng, comps, h, w, 60 + 7 * n, huff=kinds[n % 3] if n % 3 else "optimal", ri=[0, 2, 5][n % 3],
                   sof=0xC1))
    # table ids 0-3, separate per component, arbitrary component ids, no JFIF
    for n in range(6):
        ids = tuple(rng.choice(np.r_[0:82, 83:256], 3, replace=False)) if n % 2 else (0, 1, 2)
        comps = _ycc(lumas[n % 4], ids=ids, tq=(n % 4, (n + 1) % 4, (n + 2) % 4), td=(3, 2, 1 + n % 3),
                     ta=(1, 3, n % 4))
        add("ids_tables_%d" % n, _frame(rng, comps, 24 + n, 33 + 2 * n, 80, huff="long" if n % 2 else "optimal",
                                        sof=0xC1, jfif=bool(n % 3)))
    # marker layouts: tables after SOF, APPn / COM between, fill bytes, trailing bytes, 16-bit DQT
    for n in range(8):
        f = _frame(rng, _ycc(lumas[n % 4]), 30 + 3 * n, 44 - n, 85, huff=kinds[n % 3], ri=[0, 2][n % 2],
                   tables_after_sof=bool(n & 1), extras=bool(n & 2), fill=bool(n & 4), trailer=b"\x00junk" * (n % 3))
        if n >= 4:
            f.qt16 = True
        add("markers_%d" % n, f)
    # 16-bit quantisers up to 65535 where the coefficients are zero, small ones elsewhere
    for n in range(3):
        comps = _ycc((2, 2))
        f = _frame(rng, comps, 32, 48, 90, huff="optimal", qt16=True, sof=0xC1)
        for c, cf in enumerate(f.coef):
            hi = np.arange(64) >= 20 + 10 * n
            cf[..., hi] = 0
        for t in f.qt:
            f.qt[t] = np.where(np.arange(64) >= 20 + 10 * n, 65535 - 1000 * n, f.qt[t])
        add("qt16_big_%d" % n, f, legit=True)
    # sparse random blocks: ZRL runs, EOB at k = 63, every DC category 0-11
    for n in range(8):
        comps = _ycc(lumas[n % 4]) if n % 3 else [(1, 1, 1, 0, 0, 0)]
        f = _frame(rng, comps, 40, 48, 100, source="sparse", huff="optimal" if n % 2 else "long", ri=[0, 1, 4][n % 3])
        for cf in f.coef:
            cf[::2, ::2, 63] = rng.choice([-1, 1, 3], cf[::2, ::2, 63].shape)        # EOB needs no symbol after 63
        f.qt = {t: np.ones(64, np.int64) for t in f.qt}
        add("sparse_%d" % n, f, legit=False)
    # every DC category 0-11: one component in raster order, differences +-(2^c - 1) up and back down
    for n in range(2):
        f = _frame(rng, [(1, 1, 1, 0, 0, 0)], 24 + 8 * n, 64, 100, source="sparse", huff=["optimal", "long"][n])
        f.qt = {0: np.ones(64, np.int64)}
        c = np.arange(f.coef[0][..., 0].size) // 2 % 12
        f.coef[0][..., 0] = np.where(np.arange(c.size) % 2, 0, ((1 << c) - 1) * (1 - 2 * (c % 2))).reshape(
            f.coef[0].shape[:2])
        add("dc_categories_%d" % n, f, legit=False)
    # single-symbol tables: flat blocks, DC differences all zero, every block just EOB
    for n, comps in enumerate([[(1, 1, 1, 0, 0, 0)], _ycc((1, 1))]):
        f = _frame(rng, comps, 24, 40, 75, huff="single", ri=1)          # each DC difference is the DC itself
        for cf in f.coef:
            cf[:] = 0
            cf[..., 0] = 5 * (n + 1)
        add("single_symbol_%d" % n, f, legit=True)
    # progressive: libjpeg's script, custom scripts with DC successive approximation, bands, refinement
    prog_scripts = {
        "simple": SIMPLE_YCC,
        "dc_single_deep": [([0], 0, 0, 0, 3), ([1], 0, 0, 0, 2), ([2], 0, 0, 0, 0), ([0], 0, 0, 3, 2),
                           ([0], 0, 0, 2, 1), ([1], 0, 0, 2, 1), ([0], 0, 0, 1, 0), ([1], 0, 0, 1, 0),
                           ([0], 1, 9, 0, 3), ([0], 10, 63, 0, 0), ([0], 1, 9, 3, 2), ([0], 1, 9, 2, 1),
                           ([0], 1, 9, 1, 0), ([1], 1, 63, 0, 2), ([2], 1, 20, 0, 0), ([2], 21, 63, 0, 0),
                           ([1], 1, 63, 2, 1), ([1], 1, 63, 1, 0)],
        "bands": [([0, 1, 2], 0, 0, 0, 0), ([0], 1, 1, 0, 0), ([0], 2, 2, 0, 1), ([0], 3, 63, 0, 1),
                  ([0], 2, 63, 1, 0), ([1], 1, 63, 0, 0), ([2], 1, 63, 0, 0)],
    }
    for n, (name, script) in enumerate(prog_scripts.items()):
        for luma in lumas:
            h, w = [(37, 53), (16, 24), (61, 29), (9, 70)][lumas.index(luma)]
            f = _frame(rng, _ycc(luma), h, w, [75, 95, 100][n], huff=kinds[(n + lumas.index(luma)) % 3 or 1],
                       sof=0xC2, script=script, ri=[0, 1, 3, 50][lumas.index(luma)],
                       dht_per_scan=lumas.index(luma) % 2 == 1)
            add("prog_%s_%dx%d" % ((name,) + luma), f)
    for n in range(3):
        f = _frame(rng, [(1, 1, 1, 0, 0, 0)], 45, 38, [80, 100, 40][n], sof=0xC2, script=SIMPLE_GRAY, huff="long",
                   ri_per_scan=[0, 2, 5, 0, 1, 7][:] if n == 1 else None, fill=n == 2, extras=n == 2)
        add("prog_gray_%d" % n, f)
    # progressive refinement on sparse blocks with large magnitudes, correction bits in EOB runs
    for n in range(3):
        comps = _ycc(lumas[n + 1])
        f = _frame(rng, comps, 40, 56, 100, source="sparse", sof=0xC2, huff="optimal",
                   script=prog_scripts["dc_single_deep"], ri=[0, 2, 0][n], dht_per_scan=n == 2)
        f.qt = {t: np.ones(64, np.int64) for t in f.qt}
        for cf in f.coef:
            cf[..., 0] = np.clip(cf[..., 0], -1000, 1000)
        add("prog_sparse_%d" % n, f)
    # one long EOB run: 35000 blocks, almost all without AC, runs of 32767 blocks
    big = Frame(1400, 1600, [(1, 1, 1, 0, 0, 0)], [np.zeros((175, 200, 64), np.int64)], {0: np.ones(64, np.int64)},
                sof=0xC2, script=[([0], 0, 0, 0, 0), ([0], 1, 63, 0, 1), ([0], 1, 63, 1, 0)])
    big.coef[0][..., 0] = rng.randint(-300, 300, (175, 200))
    big.coef[0][0, ::37, 5] = big.coef[0][-1, ::37, 5] = 9                # runs of 173 rows between them
    add("prog_eobrun", big, legit=False)
    # ---- out of the IDCT's range: flagged on the device ----
    for n, target in enumerate([IDCT_RANGE - 1, IDCT_RANGE, IDCT_RANGE + 1, 20000, 32767, 60000]):
        comps = [(1, 1, 1, 0, 0, 0)] if n % 2 else _ycc((2, 2))
        f = _frame(rng, comps, 24, 32, 75, huff="optimal", sof=0xC1)
        f.qt = {t: np.ones(64, np.int64) for t in f.qt}
        for cf in f.coef:
            cf[:] = 0
            cf[..., 0] = rng.randint(-50, 50, cf.shape[:2])
        f.coef[0][1, 2] = boundary_block(rng, target, n % 8)
        f.coef[0][0, 0] = boundary_block(rng, min(target, IDCT_RANGE), (n + 3) % 8)
        assert int(pass1_peak(f.coef[0][1, 2], 1)) == target
        ok = all(block_in_range(cf, f.qt[c[3]]).all() for cf, c in zip(f.coef, comps))
        add("boundary_%d" % target, f, "device" if ok else "range")
    # DC-only blocks at the dequantised limit: 4095 * 4 = 16380 in pass 1, 4096 flags
    for n, dc in enumerate([4095, 4096, 8191, 8192]):
        f = _frame(rng, [(1, 1, 1, 0, 0, 0)], 16, 16, 75, huff="optimal")
        f.qt = {0: np.ones(64, np.int64)}
        f.coef[0][:] = 0
        f.coef[0][..., 0] = [[dc, -dc], [-dc, dc]]
        add("dc_only_%d" % dc, f, "device" if dc <= 4095 else "range")
    # large coefficients times large quantisers, as in hostile files
    for n in range(12):
        amp, qmax = [(60, 64), (200, 255), (100, 16), (1000, 255)][n % 4]
        comps = _ycc(lumas[n % 4])
        f = _frame(rng, comps, 24, 40, 75, source="sparse", huff="optimal", sof=0xC1, qt16=qmax > 255)
        f.coef = sparse_coefs(rng, comps, 24, 40, amp=amp, density=0.3, dc=amp)
        f.qt = {t: rng.randint(1, qmax + 1, 64) for t in f.qt}
        ok = all(block_in_range(cf, f.qt[c[3]]).all() for cf, c in zip(f.coef, comps))
        add("hostile_%d_%d_%d" % (n, amp, qmax), f, "device" if ok else "range", legit=False)
    # ---- the parser sends these to the host, or refuses them ----
    for n, key in enumerate([(0, 0), (1, 0), (0, 1), (1, 1)]):
        huff = "annexk0" if key[1] == 0 else "annexk1"
        f = _frame(rng, _ycc((2, 2)), 20, 28, 75, huff={(0, 0): "annexk0", (1, 0): "annexk0", (0, 1): "annexk1",
                                                        (1, 1): "annexk1"}, all_ones=key)
        add("all_ones_annexk_%d%d" % key, f, "raise", "prefix code")
        f = _frame(rng, _ycc((1, 1)), 20, 28, 75, huff="optimal", all_ones=key)
        add("all_ones_optimal_%d%d" % key, f, "raise", "prefix code")
        f = _frame(rng, _ycc(lumas[n]), 20, 28, 75, huff="optimal", all_ones=key, sof=0xC2, script=SIMPLE_YCC)
        add("all_ones_progressive_%d%d" % key, f, "raise", "prefix code")
    for n, (h, w) in enumerate([(8, 8), (16, 24), (33, 47), (40, 56), (64, 64), (23, 9)]):
        comps = _ycc(lumas[n % 4]) if n % 3 else [(1, 1, 1, 0, 0, 0)]
        add("no_eoi_%d" % n, _frame(rng, comps, h, w, 75, huff="optimal", eoi=False, ri=[0, 2][n % 2]), "no_eoi")
        add("no_eoi_prog_%d" % n, _frame(rng, comps, h, w, 75, huff="optimal", eoi=False, sof=0xC2,
                                         script=SIMPLE_YCC if len(comps) == 3 else SIMPLE_GRAY), "no_eoi")
    add("sampling_411", _frame(rng, _ycc((4, 1)), 24, 64, 75), "host", "sampling")
    add("sampling_chroma_21", _frame(rng, _ycc((2, 1), chroma=(2, 1)), 24, 40, 75), "host", "sampling")
    add("sampling_411_prog", _frame(rng, _ycc((4, 1)), 24, 64, 75, sof=0xC2, script=SIMPLE_YCC), "host", "sampling")
    # ---- corrupt entropy data: the parser takes the file, the device flags it ----
    for n in range(4):
        comps = _ycc(lumas[n])
        f = _frame(rng, comps, 48, 64, 90, huff={(0, 0): "annexk0", (1, 0): "annexk0", (0, 1): "annexk1",
                                                 (1, 1): "annexk1"}, ri=[0, 3][n % 2])
        add("corrupt_seq_%d" % n, corrupt_entropy(f.encode()), "corrupt")
        f = _frame(rng, comps, 48, 64, 90, huff="optimal", sof=0xC2, script=SIMPLE_YCC, ri=[0, 3][n % 2])
        add("corrupt_prog_%d" % n, corrupt_entropy(f.encode()), "corrupt")
        # cut inside the last scan's entropy data, EOI after the cut: the data ends before the last unit
        data = f.encode()
        sos = data.rindex(b"\xFF\xDA")
        add("cut_prog_%d" % n, data[:(sos + len(data)) // 2] + b"\xFF\xD9", "corrupt")
        data = _frame(rng, comps, 48, 64, 90, huff="long", ri=[0, 3][n % 2]).encode()
        sos = data.rindex(b"\xFF\xDA")
        add("cut_seq_%d" % n, data[:(sos + len(data)) // 2] + b"\xFF\xD9", "corrupt")
    return out
