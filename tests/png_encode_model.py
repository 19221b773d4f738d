"""A numpy / Python model of the device PNG encoder (csrc/png_encode.cu), stage by stage, as
``cv2.imencode('.png', img)`` writes a BGR uint8 image with OpenCV 4.13's defaults (libpng, Sub filter, zlib level 1,
strategy Z_RLE, memLevel 8):

- ``filtered(img)``: rows of filter type 1 (Sub, bpp 3) over the RGB bytes; filter type 0 (None) when the image is
  one pixel wide, since libpng drops Sub for one-pixel rows;
- ``symbols(f)``: zlib's ``deflate_rle`` parse, closed form per run of equal bytes (one literal, then matches of
  258 at distance 1, then the remainder as one match if >= 3 else as literals);
- ``deflate(f)``: blocks of 16383 symbols (``lit_bufsize - 1`` at memLevel 8) and a final block, possibly empty,
  each coded as zlib's ``_tr_flush_block`` chooses (stored / static / dynamic, ties to static) with the trees of
  ``build_tree`` (heap with the depth tie-break, ``gen_bitlen``'s repair at 15 bits, ``gen_codes``) and the
  code-length code of ``scan_tree`` / ``send_tree``;
- ``zlib_header(n)``: libpng's window reduction for at most 16 KiB of filtered data (``png_deflate_claim``) and its
  header rewrite (``optimize_cmf``);
- ``png(img)``: signature, IHDR, the zlib stream in IDAT chunks of 8192 bytes, IEND.
"""
from __future__ import annotations

import zlib

import numpy as np

BLOCK_SYMBOLS = 16383
MAX_MATCH = 258
IDAT_BYTES = 8192

L_CODES, D_CODES, BL_CODES = 286, 30, 19
HEAP_SIZE = 2 * L_CODES + 1
MAX_BITS, MAX_BL_BITS = 15, 7
END_BLOCK = 256
EXTRA_LBITS = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
BASE_LENGTH = [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 14, 16, 20, 24, 28, 32, 40, 48, 56, 64, 80, 96, 112, 128, 160, 192,
               224, 0]
# match length - 3 -> length code - 257; length 258 takes code 285, not 284 + 31
LENGTH_CODE = [max(c for c in range(28) if BASE_LENGTH[c] <= lc) for lc in range(255)] + [28]
STATIC_LLEN = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
STATIC_DLEN = [5] * D_CODES


def bi_reverse(code, n):
    r = 0
    for _ in range(n):
        r, code = (r << 1) | (code & 1), code >> 1
    return r


def gen_codes(lens, max_code, bl_count):
    next_code, code = [0] * (MAX_BITS + 1), 0
    for bits in range(1, MAX_BITS + 1):
        code = (code + bl_count[bits - 1]) << 1
        next_code[bits] = code
    codes = [0] * len(lens)
    for n in range(max_code + 1):
        if lens[n]:
            codes[n] = bi_reverse(next_code[lens[n]], lens[n])
            next_code[lens[n]] += 1
    return codes


STATIC_LCODE = gen_codes(STATIC_LLEN, 287, [0, 0, 0, 0, 0, 0, 0, 24, 152, 112, 0, 0, 0, 0, 0, 0])
STATIC_DCODE = [bi_reverse(d, 5) for d in range(D_CODES)]


def filtered(img):
    """The scanlines libpng deflates: per row the filter type byte, then Sub (or None at width 1) over RGB."""
    h, w, _ = img.shape
    rgb = np.ascontiguousarray(img[:, :, ::-1]).reshape(h, 3 * w)
    if w == 1:
        return np.concatenate([np.zeros((h, 1), np.uint8), rgb], axis=1).reshape(-1)
    sub = rgb.copy()
    sub[:, 3:] -= rgb[:, :-3]
    return np.concatenate([np.ones((h, 1), np.uint8), sub], axis=1).reshape(-1)


def symbols(f):
    """deflate_rle's symbols: v < 256 a literal, v >= 256 a match of length v - 253 at distance 1.  Computed per byte
    from the start s and end e of its run, as the device does: the byte at offset k = p - s emits a symbol iff k == 0
    (the literal), or j = k - 1 is a multiple of 258 below 258 q (a match of 258), or j >= 258 q and either r >= 3 and
    j == 258 q (a match of r) or r < 3 (a literal), where q, r = divmod(L - 1, 258)."""
    f = np.asarray(f, np.uint8)
    N = f.size
    starts = np.flatnonzero(np.r_[True, f[1:] != f[:-1]])
    lens = np.diff(np.r_[starts, N])
    s = np.repeat(starts, lens)
    L = np.repeat(lens, lens)
    k = np.arange(N) - s
    j, (q, r) = k - 1, np.divmod(L - 1, MAX_MATCH)
    full = (k > 0) & (j < MAX_MATCH * q)
    tail = (k > 0) & ~full
    emit = (k == 0) | (full & (j % MAX_MATCH == 0)) | (tail & ((r < 3) | (j == MAX_MATCH * q)))
    v = f.astype(np.int64)
    v[full] = 256 + MAX_MATCH - 3
    m = tail & (r >= 3)
    v[m] = 256 + r[m] - 3
    return v[emit]


def symbol_bytes(sym):
    return np.where(sym < 256, 1, sym - 253)


class Tree:
    """zlib's tree_desc: ``freq`` / ``lens`` / ``codes`` of the leaves, ``max_code``."""

    def __init__(self, elems, stree, extra, base, max_length):
        self.elems, self.stree, self.extra, self.base, self.max_length = elems, stree, extra, base, max_length
        self.freq = [0] * HEAP_SIZE
        self.lens = [0] * HEAP_SIZE
        self.dad = [0] * HEAP_SIZE
        self.max_code = -1
        self.codes = None


class BlockCoder:
    """One block's trees, as trees.c builds them; ``opt_len`` / ``static_len`` in bits, without the 3 header bits."""

    def __init__(self, sym):
        self.l = Tree(L_CODES, STATIC_LLEN, EXTRA_LBITS, 257, MAX_BITS)
        self.d = Tree(D_CODES, STATIC_DLEN, EXTRA_DBITS, 0, MAX_BITS)
        self.bl = Tree(BL_CODES, None, EXTRA_BLBITS, 0, MAX_BL_BITS)
        self.opt_len = self.static_len = 0
        lit = np.bincount(sym[sym < 256], minlength=256)
        lc = sym[sym >= 256] - 256
        for n in range(256):
            self.l.freq[n] = int(lit[n])
        for c, cnt in enumerate(np.bincount(np.array(LENGTH_CODE)[lc], minlength=29)):
            self.l.freq[257 + c] = int(cnt)
        self.l.freq[END_BLOCK] = 1
        self.d.freq[0] = int(lc.size)

    def smaller(self, t, n, m):
        return t.freq[n] < t.freq[m] or (t.freq[n] == t.freq[m] and self.depth[n] <= self.depth[m])

    def pqdownheap(self, t, k):
        heap, v, j = self.heap, self.heap[k], k << 1
        while j <= self.heap_len:
            if j < self.heap_len and self.smaller(t, heap[j + 1], heap[j]):
                j += 1
            if self.smaller(t, v, heap[j]):
                break
            heap[k] = heap[j]
            k, j = j, j << 1
        heap[k] = v

    def gen_bitlen(self, t):
        heap, bl_count = self.heap, [0] * (MAX_BITS + 1)
        overflow = 0
        t.lens[heap[self.heap_max]] = 0
        h = self.heap_max + 1
        while h < HEAP_SIZE:
            n = heap[h]
            bits = t.lens[t.dad[n]] + 1
            if bits > t.max_length:
                bits, overflow = t.max_length, overflow + 1
            t.lens[n] = bits
            h += 1
            if n > t.max_code:
                continue
            bl_count[bits] += 1
            xbits = t.extra[n - t.base] if n >= t.base else 0
            f = t.freq[n]
            self.opt_len += f * (bits + xbits)
            if t.stree is not None:
                self.static_len += f * (t.stree[n] + xbits)
        if overflow:
            self.overflowed = True
            while True:
                bits = t.max_length - 1
                while bl_count[bits] == 0:
                    bits -= 1
                bl_count[bits] -= 1
                bl_count[bits + 1] += 2
                bl_count[t.max_length] -= 1
                overflow -= 2
                if overflow <= 0:
                    break
            for bits in range(t.max_length, 0, -1):
                n = bl_count[bits]
                while n:
                    h -= 1
                    m = heap[h]
                    if m > t.max_code:
                        continue
                    if t.lens[m] != bits:
                        self.opt_len += (bits - t.lens[m]) * t.freq[m]
                        t.lens[m] = bits
                    n -= 1
        return bl_count

    def build_tree(self, t):
        self.heap, self.depth = [0] * HEAP_SIZE, [0] * HEAP_SIZE
        heap, self.heap_len, self.heap_max = self.heap, 0, HEAP_SIZE
        max_code = -1
        for n in range(t.elems):
            if t.freq[n]:
                self.heap_len += 1
                heap[self.heap_len] = max_code = n
            else:
                t.lens[n] = 0
        while self.heap_len < 2:
            if max_code < 2:
                max_code += 1
                node = max_code
            else:
                node = 0
            self.heap_len += 1
            heap[self.heap_len] = node
            t.freq[node] = 1
            self.opt_len -= 1
            if t.stree is not None:
                self.static_len -= t.stree[node]
        t.max_code = max_code
        for n in range(self.heap_len // 2, 0, -1):
            self.pqdownheap(t, n)
        node = t.elems
        while True:
            n = heap[1]
            heap[1] = heap[self.heap_len]
            self.heap_len -= 1
            self.pqdownheap(t, 1)
            m = heap[1]
            self.heap_max -= 1
            heap[self.heap_max] = n
            self.heap_max -= 1
            heap[self.heap_max] = m
            t.freq[node] = t.freq[n] + t.freq[m]
            self.depth[node] = max(self.depth[n], self.depth[m]) + 1
            t.dad[n] = t.dad[m] = node
            heap[1] = node
            node += 1
            self.pqdownheap(t, 1)
            if self.heap_len < 2:
                break
        self.heap_max -= 1
        heap[self.heap_max] = heap[1]
        bl_count = self.gen_bitlen(t)
        t.codes = gen_codes(t.lens, max_code, bl_count)

    def scan_tree(self, t):
        """Counts the code-length code symbols of t's lengths (0xffff past max_code is zlib's guard)."""
        for curlen, count, kind in self.runs(t):
            if kind == "lens":
                self.bl.freq[curlen] += count
            elif kind == "rep":
                if count[0]:
                    self.bl.freq[curlen] += 1
                self.bl.freq[16] += 1
            else:
                self.bl.freq[kind] += 1

    @staticmethod
    def runs(t):
        lens = t.lens[:t.max_code + 1] + [0xFFFF]
        prevlen, nextlen, count = -1, lens[0], 0
        max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
        for n in range(t.max_code + 1):
            curlen, nextlen = nextlen, lens[n + 1]
            count += 1
            if count < max_count and curlen == nextlen:
                continue
            if count < min_count:
                yield curlen, count, "lens"
            elif curlen != 0:
                yield curlen, (curlen != prevlen, count - (curlen != prevlen)), "rep"
            elif count <= 10:
                yield curlen, count, 17
            else:
                yield curlen, count, 18
            count, prevlen = 0, curlen
            if nextlen == 0:
                max_count, min_count = 138, 3
            elif curlen == nextlen:
                max_count, min_count = 6, 3
            else:
                max_count, min_count = 7, 4

    def send_tree(self, t, out):
        bl = self.bl
        for curlen, count, kind in self.runs(t):
            if kind == "lens":
                out += [(bl.codes[curlen], bl.lens[curlen])] * count
            elif kind == "rep":
                first, rest = count
                if first:
                    out.append((bl.codes[curlen], bl.lens[curlen]))
                out += [(bl.codes[16], bl.lens[16]), (rest - 3, 2)]
            elif kind == 17:
                out += [(bl.codes[17], bl.lens[17]), (count - 3, 3)]
            else:
                out += [(bl.codes[18], bl.lens[18]), (count - 11, 7)]

    def build(self):
        """build_tree for both trees, build_bl_tree; returns max_blindex."""
        self.overflowed = False
        self.build_tree(self.l)
        self.build_tree(self.d)
        self.scan_tree(self.l)
        self.scan_tree(self.d)
        self.build_tree(self.bl)
        max_blindex = BL_CODES - 1
        while max_blindex >= 3 and self.bl.lens[BL_ORDER[max_blindex]] == 0:
            max_blindex -= 1
        self.opt_len += 3 * (max_blindex + 1) + 5 + 5 + 4
        self.max_blindex = max_blindex
        return max_blindex

    def tree_bits(self):
        """send_all_trees as (value, nbits) pairs."""
        out = [(self.l.max_code + 1 - 257, 5), (self.d.max_code + 1 - 1, 5), (self.max_blindex + 1 - 4, 4)]
        out += [(self.bl.lens[BL_ORDER[r]], 3) for r in range(self.max_blindex + 1)]
        self.send_tree(self.l, out)
        self.send_tree(self.d, out)
        return out


def symbol_codes(sym, lcode, llen, dcode, dlen):
    """(value, nbits) per symbol with the literal/length code, length extra bits and distance code in one value;
    END_BLOCK appended."""
    sym = np.asarray(sym, np.int64)
    lcode, llen = np.asarray(lcode, np.int64), np.asarray(llen, np.int64)
    val, nb = lcode[np.minimum(sym, 255)].copy(), llen[np.minimum(sym, 255)].copy()
    m = sym >= 256
    lc = sym[m] - 256
    c = np.array(LENGTH_CODE)[lc]
    xb = np.array(EXTRA_LBITS)[c]
    xv = np.where(xb > 0, lc - np.array(BASE_LENGTH)[c], 0)     # code 285 (length 258) has no extra bits
    cl, cn = lcode[257 + c], llen[257 + c]
    val[m] = cl | (xv << cn) | (int(dcode[0]) << (cn + xb))
    nb[m] = cn + xb + int(dlen[0])
    return np.r_[val, lcode[END_BLOCK]], np.r_[nb, llen[END_BLOCK]]


class Bits:
    def __init__(self):
        self.vals, self.nbs, self.total = [], [], 0

    def put(self, vals, nbs):
        vals, nbs = np.atleast_1d(np.asarray(vals, np.uint64)), np.atleast_1d(np.asarray(nbs, np.int64))
        self.vals.append(vals)
        self.nbs.append(nbs)
        self.total += int(nbs.sum())

    def align(self):
        self.put(0, (-self.total) % 8)

    def bytes(self):
        self.align()
        vals, nbs = np.concatenate(self.vals), np.concatenate(self.nbs)
        idx = np.repeat(np.arange(vals.size), nbs)
        pos = np.arange(self.total) - np.repeat(np.cumsum(nbs) - nbs, nbs)
        bits = ((vals[idx] >> pos.astype(np.uint64)) & np.uint64(1)).astype(np.uint8)
        return np.packbits(bits, bitorder="little").tobytes()


def block_choice(coder, stored_len, in_window=True):
    """_tr_flush_block's choice: 'stored', 'static' or 'dynamic'."""
    opt_lenb = (coder.opt_len + 3 + 7) >> 3
    static_lenb = (coder.static_len + 3 + 7) >> 3
    opt_lenb = min(opt_lenb, static_lenb)
    if stored_len + 4 <= opt_lenb and in_window:
        return "stored"
    return "static" if static_lenb == opt_lenb else "dynamic"


def deflate(f, trace=None):
    """The raw deflate data of f as zlib writes it at these settings.  ``trace``, a list, receives one
    ``(kind, nsym, stored_len, coder)`` per block."""
    f = np.asarray(f, np.uint8)
    sym = symbols(f)
    nblocks = sym.size // BLOCK_SYMBOLS + 1
    out, pos = Bits(), 0
    for b in range(nblocks):
        s = sym[b * BLOCK_SYMBOLS:(b + 1) * BLOCK_SYMBOLS]
        last = int(b == nblocks - 1)
        stored_len = int(symbol_bytes(s).sum())
        coder = BlockCoder(s)
        coder.build()
        kind = block_choice(coder, stored_len)
        if trace is not None:
            trace.append((kind, s.size, stored_len, coder))
        if kind == "stored":
            out.put(last, 3)
            out.align()
            out.put([stored_len & 0xFFFF, ~stored_len & 0xFFFF], [16, 16])
            out.put(f[pos:pos + stored_len], np.full(stored_len, 8))
        elif kind == "static":
            out.put(2 + last, 3)
            out.put(*symbol_codes(s, STATIC_LCODE, STATIC_LLEN, STATIC_DCODE, STATIC_DLEN))
        else:
            out.put(4 + last, 3)
            tb = coder.tree_bits()
            out.put([v for v, _ in tb], [n for _, n in tb])
            out.put(*symbol_codes(s, coder.l.codes, coder.l.lens, coder.d.codes, coder.d.lens))
        pos += stored_len
    return out.bytes()


def window_bits(n):
    """png_deflate_claim: at most 16 KiB of data lowers windowBits while n + 262 fits in half the window."""
    wb = 15
    if n <= 16384:
        half = 1 << (wb - 1)
        while n + 262 <= half:
            half >>= 1
            wb -= 1
    return wb


def zlib_header(n):
    """The two header bytes: zlib's for window_bits(n) at level 1, then libpng's optimize_cmf rewrite."""
    cmf = ((window_bits(n) - 8) << 4) | 8
    if n <= 16384:
        cinfo = cmf >> 4
        half = 1 << (cinfo + 7)
        if n <= half:
            while True:
                half >>= 1
                cinfo -= 1
                if not (cinfo > 0 and n <= half):
                    break
            cmf = (cinfo << 4) | 8
    return bytes([cmf, 31 - (cmf << 8) % 31])


def adler32(f):
    f = np.asarray(f, np.uint8).astype(np.int64)
    n = f.size
    s1 = (1 + int(f.sum())) % 65521
    s2 = (n + int((f * (n - np.arange(n))).sum() % 65521)) % 65521
    return (s2 << 16) | s1


def zstream(img):
    f = filtered(img)
    return zlib_header(f.size) + deflate(f) + adler32(f).to_bytes(4, "big")


def chunk(kind, data):
    return len(data).to_bytes(4, "big") + kind + data + zlib.crc32(kind + data).to_bytes(4, "big")


def png(img):
    """The file cv2.imencode('.png', img) writes for a BGR uint8 (H, W, 3) image."""
    h, w, _ = img.shape
    z = zstream(img)
    ihdr = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr)
    for i in range(0, len(z), IDAT_BYTES):
        out += chunk(b"IDAT", z[i:i + IDAT_BYTES])
    return out + chunk(b"IEND", b"")
