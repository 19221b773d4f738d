"""A test-only VP8 key-frame writer (RFC 6386) with a boolean encoder.  It writes chosen syntax elements directly, with
no rate-distortion search: header fields (segmentation, loop filter and its deltas, partitions, quantiser indices and
deltas, coefficient-probability updates, skip probability) and per macroblock its segment, skip flag, intra modes and
quantised coefficient levels.  So every branch of a decoder can be reached on purpose, which cv2.imencode, which only
exposes a quality, cannot do.  ``Frame.encode()`` returns a simple-container WebP file; ``matrix()`` builds the
test matrix's frames from a seed.  4x4 modes are numbered as libwebp does: DC, TM, VE, HE, RD, VR, LD, VL, HD, HU."""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

from tests import vp8_tables

B_DC, B_TM, B_VE, B_HE, B_RD, B_VR, B_LD, B_VL, B_HD, B_HU = range(10)
BANDS = (0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0)
ZIGZAG = (0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15)
CAT3456 = ((173, 148, 140), (176, 155, 140, 135), (180, 157, 141, 134, 130),
           (254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129))
MODE_TREE = (-B_DC, 1, -B_TM, 2, -B_VE, 3, 4, 6, -B_HE, 5, -B_RD, -B_VR, -B_LD, 7, -B_VL, 8, -B_HD, -B_HU)
UPDATE = np.array(vp8_tables.COEFFS_UPDATE_PROBA).reshape(4, 8, 3, 11)
PROBA0 = np.array(vp8_tables.COEFFS_PROBA0).reshape(4, 8, 3, 11)
BMODES = np.array(vp8_tables.BMODES_PROBA).reshape(10, 10, 9)
MAX_LEVEL = 2048 + 66                      # the largest DCT_CAT6 token


def _mode_paths():
    """mode -> [(tree node, bit)] of the 4x4 mode tree (node i reads prob[i] and goes to MODE_TREE[2 i + bit])."""
    paths = {}

    def walk(node, path):
        for b in (0, 1):
            nxt = MODE_TREE[2 * node + b]
            if nxt > 0:
                walk(nxt, path + [(node, b)])
            else:
                paths[-nxt] = path + [(node, b)]
    walk(0, [])
    return paths


MODE_PATHS = _mode_paths()


class BoolEncoder:
    """RFC 6386 7.3's boolean encoder."""

    def __init__(self):
        self.out = bytearray()
        self.range, self.bottom, self.bit_count = 255, 0, 24

    def put(self, bit, prob):
        split = 1 + (((self.range - 1) * prob) >> 8)
        if bit:
            self.bottom += split
            self.range -= split
        else:
            self.range = split
        while self.range < 128:
            self.range <<= 1
            if self.bottom & (1 << 31):
                i = len(self.out) - 1
                while self.out[i] == 255:
                    self.out[i] = 0
                    i -= 1
                self.out[i] += 1
            self.bottom = (self.bottom << 1) & 0xFFFFFFFF
            self.bit_count -= 1
            if not self.bit_count:
                self.out.append(self.bottom >> 24)
                self.bottom &= (1 << 24) - 1
                self.bit_count = 8

    def literal(self, v, n):
        for k in range(n - 1, -1, -1):
            self.put((v >> k) & 1, 128)

    def signed(self, v, n):
        self.literal(abs(v), n)
        self.put(v < 0, 128)

    def flagged(self, v, n):
        """A flag and, when ``v`` is not None, a signed n-bit value."""
        self.put(v is not None, 128)
        if v is not None:
            self.signed(v, n)

    def flush(self):
        for _ in range(32):
            self.put(0, 128)
        return bytes(self.out)


@dataclass
class Macroblock:
    segment: int = 0
    skip: int = 0                          # the coded skip flag (used when the frame has a skip probability)
    i4x4: bool = False
    ymode: int = B_DC                      # 16x16 mode: B_DC, B_TM, B_VE or B_HE
    imodes: list = field(default_factory=lambda: [B_DC] * 16)
    uvmode: int = B_DC
    # quantised levels in zigzag order: 16 luma, 4 U, 4 V blocks, then the Y2 block (16x16 modes only)
    levels: np.ndarray = field(default_factory=lambda: np.zeros((25, 16), np.int64))


@dataclass
class Frame:
    w: int
    h: int
    mbs: list                              # row-major macroblocks
    use_segment: bool = False
    update_map: bool = False
    update_data: bool = False
    absolute: bool = True
    seg_quant: tuple = (None,) * 4         # None: flag off (0)
    seg_filter: tuple = (None,) * 4
    seg_probs: tuple = (None,) * 3         # None: not sent (255)
    simple: bool = False
    level: int = 20
    sharpness: int = 0
    use_lf_delta: bool = False
    update_lf_delta: bool = False
    ref_deltas: tuple = (None,) * 4
    mode_deltas: tuple = (None,) * 4
    log2_parts: int = 0
    q0: int = 40
    dq: dict = field(default_factory=dict)  # y1dc, y2dc, y2ac, uvdc, uvac -> delta (-15..15)
    proba_updates: dict = field(default_factory=dict)  # (t, b, c, p) -> probability
    skip_prob: int = None                  # None: no skip probability

    def steps(self, segment):
        """The dequantisation steps (y1 dc, y1 ac, y2 dc, y2 ac, uv dc, uv ac) of ``segment`` (RFC 6386 9.6, 14.1)."""
        q = self.q0
        if self.use_segment:                  # without a data update the segment values stay 0, absolute
            q = (self.seg_quant[segment] or 0) if self.update_data else 0
            if self.update_data and not self.absolute:
                q += self.q0
        dc, ac = vp8_tables.DC_TABLE, vp8_tables.AC_TABLE
        clip = lambda v, m: min(max(v, 0), m)
        d = lambda k: self.dq.get(k) or 0
        y2ac = ac[clip(q + d("y2ac"), 127)] * 155 // 100
        return (dc[clip(q + d("y1dc"), 127)], ac[clip(q, 127)], 2 * dc[clip(q + d("y2dc"), 127)], max(y2ac, 8),
                dc[clip(q + d("uvdc"), 117)], ac[clip(q + d("uvac"), 127)])

    def legalize(self):
        """Clip every level so that its dequantised coefficient lies in RFC 6386's range: +-2047 for the DCT blocks,
        +-1023 for the Y2 block, whose inverse WHT doubles the range of the luma DCs it makes.  libwebp's SIMD
        transforms, which cv2 runs, assume that range."""
        for mb in self.mbs:
            y1dc, y1ac, y2dc, y2ac, uvdc, uvac = self.steps(mb.segment)
            for b, (dc, ac, m) in ((slice(0, 16), (y1dc, y1ac, 2047)), (slice(16, 24), (uvdc, uvac, 2047)),
                                   (slice(24, 25), (y2dc, y2ac, 1023))):
                mb.levels[b, 0] = np.clip(mb.levels[b, 0], -(m // dc), m // dc)
                mb.levels[b, 1:] = np.clip(mb.levels[b, 1:], -(m // ac), m // ac)
        return self

    def probas(self):
        p = PROBA0.copy()
        for k, v in self.proba_updates.items():
            p[k] = v
        return p

    def encode(self):
        mbw, mbh = (self.w + 15) >> 4, (self.h + 15) >> 4
        assert len(self.mbs) == mbw * mbh
        e = BoolEncoder()
        e.put(0, 128)                      # colour space
        e.put(0, 128)                      # clamping type
        e.put(self.use_segment, 128)
        if self.use_segment:
            e.put(self.update_map, 128)
            e.put(self.update_data, 128)
            if self.update_data:
                e.put(self.absolute, 128)
                for v in self.seg_quant:
                    e.flagged(v, 7)
                for v in self.seg_filter:
                    e.flagged(v, 6)
            if self.update_map:
                for v in self.seg_probs:
                    e.put(v is not None, 128)
                    if v is not None:
                        e.literal(v, 8)
        e.put(self.simple, 128)
        e.literal(self.level, 6)
        e.literal(self.sharpness, 3)
        e.put(self.use_lf_delta, 128)
        if self.use_lf_delta:
            e.put(self.update_lf_delta, 128)
            if self.update_lf_delta:
                for v in self.ref_deltas + self.mode_deltas:
                    e.flagged(v, 6)
        e.literal(self.log2_parts, 2)
        e.literal(self.q0, 7)
        for k in ("y1dc", "y2dc", "y2ac", "uvdc", "uvac"):
            e.flagged(self.dq.get(k), 4)
        e.put(0, 128)                      # refresh_entropy_probs
        probas = self.probas()
        for idx in np.ndindex(4, 8, 3, 11):
            upd = idx in self.proba_updates
            e.put(upd, int(UPDATE[idx]))
            if upd:
                e.literal(int(probas[idx]), 8)
        e.put(self.skip_prob is not None, 128)
        if self.skip_prob is not None:
            e.literal(self.skip_prob, 8)
        seg_p = [255 if v is None else v for v in self.seg_probs]
        intra_t = [B_DC] * (4 * mbw)
        for y in range(mbh):
            intra_l = [B_DC] * 4
            for x in range(mbw):
                mb = self.mbs[y * mbw + x]
                if self.update_map:
                    e.put(mb.segment >= 2, seg_p[0])
                    e.put(mb.segment & 1, seg_p[1 + (mb.segment >= 2)])
                if self.skip_prob is not None:
                    e.put(mb.skip, self.skip_prob)
                e.put(not mb.i4x4, 145)
                if not mb.i4x4:
                    m = mb.ymode
                    e.put(m in (B_TM, B_HE), 156)
                    e.put(m in (B_TM, B_VE), 128 if m in (B_TM, B_HE) else 163)
                    intra_t[4 * x:4 * x + 4] = [m] * 4
                    intra_l = [m] * 4
                else:
                    for sy in range(4):
                        for sx in range(4):
                            m = mb.imodes[4 * sy + sx]
                            prob = BMODES[intra_t[4 * x + sx], intra_l[sy]]
                            for node, b in MODE_PATHS[m]:
                                e.put(b, int(prob[node]))
                            intra_t[4 * x + sx] = intra_l[sy] = m
                m = mb.uvmode
                e.put(m != B_DC, 142)
                if m != B_DC:
                    e.put(m != B_VE, 114)
                    if m != B_VE:
                        e.put(m == B_TM, 183)
        part0 = e.flush()
        parts = [BoolEncoder() for _ in range(1 << self.log2_parts)]
        nz_dc_t = [0] * mbw
        nz_t = [[0] * 8 for _ in range(mbw)]                          # per column: 4 Y, 2 U, 2 V
        for y in range(mbh):
            t = parts[y % len(parts)]
            nz_l, nz_dc_l = [0] * 8, 0
            for x in range(mbw):
                mb = self.mbs[y * mbw + x]
                if self.skip_prob is not None and mb.skip:
                    nz_t[x] = [0] * 8
                    nz_l = [0] * 8
                    if not mb.i4x4:
                        nz_dc_t[x] = nz_dc_l = 0
                    continue
                first = 0
                if not mb.i4x4:
                    nz = _put_coeffs(t, probas[1], nz_dc_t[x] + nz_dc_l, 0, mb.levels[24])
                    nz_dc_t[x] = nz_dc_l = int(nz > 0)
                    first = 1
                ytype = 0 if not mb.i4x4 else 3
                top, left = nz_t[x], nz_l
                for b in range(16):
                    sy, sx = b >> 2, b & 3
                    nz = _put_coeffs(t, probas[ytype], top[sx] + left[sy], first, mb.levels[b])
                    top[sx] = left[sy] = int(nz > first)
                for c in range(2):
                    for b in range(4):
                        sy, sx = b >> 1, b & 1
                        k = 4 + 2 * c
                        nz = _put_coeffs(t, probas[2], top[k + sx] + left[k + sy], 0, mb.levels[16 + 4 * c + b])
                        top[k + sx] = left[k + sy] = int(nz > 0)
                nz_t[x], nz_l = top, left
        tokens = [p.flush() for p in parts]
        tag = (1 << 4) | (len(part0) << 5)
        vp8 = struct.pack("<I", tag)[:3] + b"\x9d\x01\x2a" + struct.pack("<HH", self.w, self.h) + part0
        vp8 += b"".join(struct.pack("<I", len(p))[:3] for p in tokens[:-1]) + b"".join(tokens)
        body = b"VP8 " + struct.pack("<I", len(vp8)) + vp8 + (b"\0" if len(vp8) & 1 else b"")
        return b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WEBP" + body


def _put_coeffs(e, P, ctx, first, lv):
    """The tokens of one block's levels (zigzag order) from position ``first``; returns the decoder's "nz" (the
    position after the last non-zero level, ``first`` when there is none)."""
    nzs = [n for n in range(first, 16) if lv[n]]
    last = nzs[-1] if nzs else -1
    n = first
    p = P[BANDS[n], ctx]
    while n < 16:
        if n > last:
            e.put(0, int(p[0]))
            return n
        e.put(1, int(p[0]))
        while lv[n] == 0:
            e.put(0, int(p[1]))
            n += 1
            p = P[BANDS[n], 0]
        e.put(1, int(p[1]))
        v = abs(int(lv[n]))
        if v == 1:
            e.put(0, int(p[2]))
            ctx = 1
        else:
            e.put(1, int(p[2]))
            _put_large(e, p, v)
            ctx = 2
        e.put(lv[n] < 0, 128)
        n += 1
        p = P[BANDS[n], ctx]
    return 16


def _put_large(e, p, v):
    if v <= 4:
        e.put(0, int(p[3]))
        e.put(v > 2, int(p[4]))
        if v > 2:
            e.put(v - 3, int(p[5]))
    elif v <= 10:
        e.put(1, int(p[3]))
        e.put(0, int(p[6]))
        e.put(v > 6, int(p[7]))
        if v <= 6:
            e.put(v - 5, 159)
        else:
            e.put((v - 7) >> 1, 165)
            e.put((v - 7) & 1, 145)
    else:
        e.put(1, int(p[3]))
        e.put(1, int(p[6]))
        cat = next(c for c in range(4) if c == 3 or v < 3 + (8 << (c + 1)))
        e.put(cat >> 1, int(p[8]))
        e.put(cat & 1, int(p[9 + (cat >> 1)]))
        extra, tab = v - 3 - (8 << cat), CAT3456[cat]
        for k, prob in enumerate(tab):
            e.put((extra >> (len(tab) - 1 - k)) & 1, prob)


def random_macroblocks(w, h, rng, segments=1, skip_rate=0.2, i4x4_rate=0.5, big_rate=0.05, density=0.3,
                       cover=None):
    """Macroblocks with random modes and sparse random levels (some up to the largest token).  ``cover``, a dict, picks
    each 4x4 mode as the one least used so far under its (above, left) context, to reach every context."""
    mbw, mbh = (w + 15) >> 4, (h + 15) >> 4
    intra_t = [B_DC] * (4 * mbw)
    out = []
    for y in range(mbh):
        intra_l = [B_DC] * 4
        for x in range(mbw):
            mb = Macroblock(segment=int(rng.integers(segments)), skip=int(rng.random() < skip_rate),
                            i4x4=bool(rng.random() < i4x4_rate), ymode=int(rng.choice([B_DC, B_TM, B_VE, B_HE])),
                            uvmode=int(rng.choice([B_DC, B_TM, B_VE, B_HE])))
            if mb.i4x4:
                for sy in range(4):
                    for sx in range(4):
                        a, l = intra_t[4 * x + sx], intra_l[sy]
                        if cover is not None:
                            m = min(range(10), key=lambda m: (cover.get((a, l, m), 0), rng.random()))
                            cover[(a, l, m)] = cover.get((a, l, m), 0) + 1
                        else:
                            m = int(rng.integers(10))
                        mb.imodes[4 * sy + sx] = m
                        intra_t[4 * x + sx] = intra_l[sy] = m
            else:
                intra_t[4 * x:4 * x + 4] = [mb.ymode] * 4
                intra_l = [mb.ymode] * 4
            lv = np.where(rng.random((25, 16)) < density, rng.integers(-12, 13, (25, 16)), 0)
            big = rng.random((25, 16)) < big_rate
            lv[big] = rng.integers(-MAX_LEVEL, MAX_LEVEL + 1, int(big.sum()))
            if mb.i4x4:
                lv[24] = 0
            else:
                lv[:16, 0] = 0                 # the luma DCs come from the Y2 block
            mb.levels = lv
            out.append(mb)
    return out


SIZES = [(1, 1), (1, 17), (17, 1), (15, 17), (16, 16), (17, 33), (130, 3), (3, 130)]   # (h, w)


def matrix():
    """(name, Frame) pairs that reach every branch of the decoder: both filter types at levels 0, 1 and 63 and every
    sharpness; reference and mode loop-filter deltas; 1-4 segments with absolute and relative values, map updates with
    and without tree probabilities, segmentation without a map or a data update; 1, 2, 4 and 8 token partitions
    (more partitions than macroblock rows too); coefficient-probability updates; skip probability on and off; every 4x4
    mode under every above / left context and all 16x16 and chroma modes, at the frame's edges; quantiser indices 0
    and 127 with every delta.  Seeded, the same on every call."""
    rng = np.random.default_rng(6386)
    out = []

    def add(name, h, w, mb_kw=None, **kw):
        out.append((name, Frame(w, h, random_macroblocks(w, h, rng, **(mb_kw or {})), **kw).legalize()))

    for h, w in SIZES:
        add("size %dx%d" % (h, w), h, w)
    for simple in (False, True):
        for level in (0, 1, 63):
            add("simple %d level %d" % (simple, level), 33, 40, simple=simple, level=level)
        for sharp in range(8):
            add("simple %d sharpness %d" % (simple, sharp), 40, 33, simple=simple, level=12 + 7 * sharp,
                sharpness=sharp)
        add("simple %d deltas" % simple, 33, 48, simple=simple, level=30, use_lf_delta=True, update_lf_delta=True,
            ref_deltas=(-20, 5, None, 63 - 126), mode_deltas=(25, None, -3, 9))
    add("deltas clamp to 63", 33, 48, level=50, use_lf_delta=True, update_lf_delta=True, ref_deltas=(30, None,) * 2,
        mode_deltas=(40, None, None, None))
    add("deltas clamp to 0", 33, 48, level=5, use_lf_delta=True, update_lf_delta=True, ref_deltas=(-30, None) * 2,
        mode_deltas=(-40, None, None, None))
    add("lf delta flag without update", 33, 48, level=25, use_lf_delta=True)
    for nseg in (1, 2, 3, 4):
        for absolute in (True, False):
            q = (10, 90, None, 127) if absolute else (-20, 15, None, 60)
            f = (40, None, 0, 63) if absolute else (-10, 25, None, 30)
            add("segments %d absolute %d" % (nseg, absolute), 48, 50, {"segments": nseg}, level=20, q0=40,
                use_segment=True, update_map=True, update_data=True, absolute=absolute, seg_quant=q, seg_filter=f,
                seg_probs=(90, None, 200) if nseg > 2 else (None, 60, None))
    add("segment map without data update", 40, 40, {"segments": 4}, use_segment=True, update_map=True,
        seg_probs=(128, 128, 128))
    add("segment data without map", 40, 40, use_segment=True, update_data=True, absolute=False,
        seg_quant=(30, -40, 0, 0), seg_filter=(-15, 0, 0, 20))
    add("segmentation without updates", 40, 40, use_segment=True)
    for log2 in range(4):
        add("partitions %d" % (1 << log2), 130, 20, log2_parts=log2)
        add("partitions %d, 2 rows" % (1 << log2), 17, 40, log2_parts=log2)
    updates = {idx: int(rng.integers(1, 256)) for idx in np.ndindex(4, 8, 3, 11) if rng.random() < 0.15}
    add("probability updates", 48, 48, proba_updates=updates)
    add("skip probability", 48, 48, {"skip_rate": 0.4}, skip_prob=100)
    add("skip probability, all skipped", 32, 48, {"skip_rate": 1.0}, skip_prob=3)
    add("no skip probability", 48, 48, {"skip_rate": 0.6})
    cover = {}
    for k in range(2):
        add("4x4 mode contexts %d" % k, 128, 160, {"i4x4_rate": 1.0, "cover": cover, "density": 0.1})
    add("16x16 and chroma modes at the edges", 48, 64, {"i4x4_rate": 0.0})
    for q0 in (0, 127):
        for k in ("y1dc", "y2dc", "y2ac", "uvdc", "uvac"):
            for d in (-15, 15):
                add("q %d %s %+d" % (q0, k, d), 17, 33, q0=q0, dq={k: d})
        add("q %d all deltas" % q0, 33, 17, q0=q0, dq={"y1dc": 7, "y2dc": -9, "y2ac": 15, "uvdc": -15, "uvac": 3})
    return out
