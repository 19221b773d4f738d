"""Host side of the device JPEG decoder (``cpb200_jpeg_decode_batch``, ``csrc/jpeg.cu``).

``parse(data, name)`` reads a file's headers and decides whether the device can decode it byte for byte as
``cv2.imread(path, IMREAD_COLOR)`` does (libjpeg-turbo's Huffman decoders, ISLOW IDCT, fancy upsampling, integer
YCbCr->BGR, then OpenCV's EXIF orientation).  ``pack(...)`` lays out the device table of a launch.

The device decodes 8-bit grayscale or YCbCr files with chroma sampled (1, 1) and luma (1, 1), (2, 1), (1, 2) or
(2, 2), in one of two forms, which ``parse`` reports as a pair:

- ``info.eligible``: sequential Huffman (SOF0 / SOF1), one interleaved scan over every component.  The sequential
  entropy kernel decodes it.
- ``info.progressive``: progressive Huffman (SOF2), the list of its scans (``JpegScan``).  The progressive entropy
  kernel decodes it.  The scans must be legal (T.81 G.1.1.1) and consistent (each scan sends coefficient bits not sent
  before, or refines the bit the previous scan stopped at; no AC scan before its component's first DC scan), at most
  ``MAX_SCANS``, with no DQT or other frame marker between them, and must code every coefficient down to bit 0 by the
  end of the file.  With an incomplete progression libjpeg smooths the low-frequency coefficients of each block
  (``jdcoefct.c``), which the device does not do.

Everything else has ``eligible == False`` and ``progressive is None``, ``reason`` says why, and the file stays with
``cv2.imread``.  The kernels trust the table, so everything read from the file that sizes or indexes it is checked
here; a file the parser cannot read raises ``ValueError`` naming the image.  That includes a Huffman table with an
all-ones code, which libjpeg refuses.

The device sets status 1 for a file it takes, which then goes to ``cv2.imread``, when:

- its last scan is not ended by EOI (``info.eoi`` False, the table's ``missing_eoi``).  libjpeg refuses some such
  files and reads others, by more than their headers say, so the kernels do not decode them.
- its entropy data ends early or holds an undefined code.
- a block's dequantised coefficients or IDCT pass-1 outputs leave +-``IDCT_RANGE``.  There libjpeg-turbo's 16-bit SIMD
  arithmetic saturates or wraps, and no real encoder goes.
"""
from __future__ import annotations

import numpy as np

# the C ABI entry point that decodes a launch packed by pack()
KERNEL = "jpeg_decode_batch"
# zigzag index -> natural (row-major) index, T.81 figure A.6
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)
LUT_BITS = 9
# jpeg_idct_kernel sets status 1 for a block with a dequantised coefficient or a pass-1 output beyond +-IDCT_RANGE:
# below it every sum and product libjpeg-turbo's 16-bit SIMD IDCT forms fits int16 (see DESIGN.md)
IDCT_RANGE = 16383
# libjpeg refuses dimensions above JPEG_MAX_DIMENSION, so cv2.imread returns nothing for them: they stay on the host
MAX_DIMENSION = 65500

# struct cpb200_jpeg_huff (include/centerpose_b200.h): a 9-bit lookup (code length << 8 | symbol, 0 = longer code),
# then T.81 F.2.2.3's maxcode / (valptr - mincode) per code length 0..17 and the symbols
HUFF = np.dtype([("lut", "<u2", (1 << LUT_BITS,)), ("maxcode", "<i4", (18,)), ("valoff", "<i4", (18,)),
                 ("val", "u1", (256,))])
assert HUFF.itemsize == 1424
# struct cpb200_jpeg_image (include/centerpose_b200.h)
JPEG_IMAGE = np.dtype([("seg_offset", "<i8"), ("huff_offset", "<i8"), ("coef_offset", "<i8"), ("plane_offset", "<i8"),
                       ("dst_offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("ncomp", "<i4"), ("hs", "<i4"), ("vs", "<i4"),
                       ("orientation", "<i4"), ("restart_interval", "<i4"), ("nseg", "<i4"), ("dc_tbl", "u1", (4,)),
                       ("ac_tbl", "u1", (4,)), ("qt", "<u2", (3, 64)), ("scan_offset", "<i8"), ("nscan", "<i4"),
                       ("missing_eoi", "<i4")])
assert JPEG_IMAGE.itemsize == 480
# struct cpb200_jpeg_scan (include/centerpose_b200.h): one scan of a progressive image
SCAN = np.dtype([("seg_offset", "<i8"), ("nseg", "<i4"), ("restart_interval", "<i4"), ("ncomp", "<i4"),
                 ("comp", "u1", (4,)), ("dc_tbl", "u1", (4,)), ("ac_tbl", "u1", (4,)), ("ss", "u1"), ("se", "u1"),
                 ("ah", "u1"), ("al", "u1"), ("pad", "<i4")])
assert SCAN.itemsize == 40
# scans per progressive file the device takes (libjpeg's simple progression writes 10 for colour, 6 for grayscale)
MAX_SCANS = 64


class JpegInfo:
    """What ``parse`` found.  ``eligible`` says whether the device decodes the file (``reason`` says why not).  For
    eligible files: ``h, w`` the coded size, ``oh, ow`` the size after the EXIF ``orientation`` (what ``cv2.imread``
    returns), ``ncomp``, luma sampling ``hs, vs``, per component quantisation tables (natural order, ``qt``) and
    Huffman table numbers (``dc``, ``ac``), the tables themselves (``huff[(class, id)]`` = (bits, values, ``HUFF``)),
    ``restart_interval`` and ``segments``, the (start, end) byte range of each entropy-coded segment.  For progressive
    files the device takes, ``progressive`` is the list of scans (``JpegScan``) and ``tables`` the ``HUFF`` tables
    they bind, in the order of their first use; ``qt`` is set, and ``dc``, ``ac``, ``restart_interval`` and
    ``segments`` are per scan.  ``eoi`` says whether EOI ends the last scan (the device flags the file otherwise)."""

    def __init__(self):
        self.eligible = False
        self.progressive = None
        self.reason = ""
        self.orientation = 1
        self.restart_interval = 0
        self.eoi = True

    def size_after_orientation(self):
        return oriented_size(self.h, self.w, self.orientation)

    @property
    def mcu(self):
        """MCUs per row and per column."""
        return -(-self.w // (8 * self.hs)), -(-self.h // (8 * self.vs))

    def blocks(self):
        """(blocks per row, block rows) of each component in the coefficient workspace: whole MCUs."""
        mx, my = self.mcu
        return [(mx * self.hs, my * self.vs)] + [(mx, my)] * (self.ncomp - 1)

    def workspace_bytes(self):
        """int16 coefficients (128 bytes per block) and 8-bit planes (64 bytes per block)."""
        return sum(bw * bh for bw, bh in self.blocks()) * 192

    def coded_blocks(self, c):
        """(blocks per row, block rows) that a scan of component ``c`` alone covers: its own samples, not whole MCUs
        (T.81 A.2.2)."""
        hs, vs = (self.hs, self.vs) if c == 0 else (1, 1)
        cw, ch = -(-self.w * hs // self.hs), -(-self.h * vs // self.vs)
        return -(-cw // 8), -(-ch // 8)


class JpegScan:
    """One scan of a progressive file: component indices ``comps`` (frame order), spectral selection ``ss..se``,
    successive approximation ``ah, al``, per component the index in ``JpegInfo.tables`` of its DC table (``dc``, for a
    first DC scan) and AC table (``ac``, for an AC scan), 0 where the scan uses none, ``restart_interval`` (units: MCUs
    for several components, blocks of ``coded_blocks`` for one) and ``segments`` as for sequential files."""

    def __init__(self, comps, ss, se, ah, al, dc, ac, restart_interval, segments):
        self.comps, self.ss, self.se, self.ah, self.al = comps, ss, se, ah, al
        self.dc, self.ac, self.restart_interval, self.segments = dc, ac, restart_interval, segments

    def units(self, info):
        """Units the scan codes: MCUs when it interleaves components, else the component's blocks."""
        if len(self.comps) > 1:
            mx, my = info.mcu
            return mx * my
        bw, bh = info.coded_blocks(self.comps[0])
        return bw * bh


def oriented_size(h, w, orientation):
    """(height, width) of an ``h`` x ``w`` image after OpenCV applies EXIF ``orientation`` (5..8 transpose it)."""
    return (w, h) if orientation >= 5 else (h, w)


def _exif_orientation(seg):
    """The orientation tag (0x0112) of IFD0 in an APP1 Exif payload, 1 when absent or unreadable."""
    if len(seg) < 14 or seg[:6] != b"Exif\x00\x00":
        return 1
    return tiff_orientation(seg[6:])


def tiff_orientation(t):
    """The orientation tag (0x0112) of IFD0 in Exif data that starts with its TIFF header (the payload of a PNG eXIf
    chunk, or of a JPEG APP1 segment after ``Exif\\0\\0``), 1 when absent or unreadable."""
    if len(t) < 8:
        return 1
    if t[:2] == b"II":
        order = "<"
    elif t[:2] == b"MM":
        order = ">"
    else:
        return 1
    u16 = lambda o: int(np.frombuffer(t, order + "u2", 1, o)[0])
    u32 = lambda o: int(np.frombuffer(t, order + "u4", 1, o)[0])
    ifd = u32(4)
    if ifd + 2 > len(t):
        return 1
    for n in range(u16(ifd)):
        e = ifd + 2 + 12 * n
        if e + 12 > len(t):
            return 1
        if u16(e) == 0x0112:
            v = u16(e + 8)
            return v if 1 <= v <= 8 else 1
    return 1


def build_huff(bits, vals, name, dc):
    """One ``HUFF`` table from the DHT code-length counts ``bits[1..16]`` and symbols; rejects counts that do not form
    a prefix code without an all-ones code (T.81 C.2, Annex C: no code may consist of 1-bits only) and, for DC tables,
    symbols above 15 (libjpeg refuses all of these)."""
    if sum(bits) > 256 or sum(bits) > len(vals):
        raise ValueError("%s: bad Huffman table (%d codes)" % (name, sum(bits)))
    if dc and any(v > 15 for v in vals):
        raise ValueError("%s: DC Huffman symbol above 15" % name)
    t = np.zeros((), HUFF)
    t["maxcode"][:] = -1
    t["maxcode"][17] = 0x7FFFFFFF
    t["val"][:len(vals)] = vals
    code, k = 0, 0
    for ln in range(1, 17):
        n = bits[ln - 1]
        if n:
            t["valoff"][ln] = k - code
            for _ in range(n):
                if ln <= LUT_BITS:
                    lo = code << (LUT_BITS - ln)
                    t["lut"][lo:lo + (1 << (LUT_BITS - ln))] = (ln << 8) | vals[k]
                code += 1
                k += 1
            t["maxcode"][ln] = code - 1
        if code >= (1 << ln):                    # the next code of this length would be all ones, or no code fits
            raise ValueError("%s: Huffman code lengths do not form a prefix code without an all-ones code" % name)
        code <<= 1
    return t


def _read_dht(seg, huff, name):
    """The tables of one DHT payload into ``huff[(class, id)]``."""
    o = 0
    while o < len(seg):
        if o + 17 > len(seg):
            raise ValueError("%s: bad Huffman table" % name)
        tc, th = seg[o] >> 4, seg[o] & 15
        bits = list(seg[o + 1:o + 17])
        cnt = sum(bits)
        if tc > 1 or th > 3 or o + 17 + cnt > len(seg):
            raise ValueError("%s: bad Huffman table" % name)
        vals = list(seg[o + 17:o + 17 + cnt])
        huff[(tc, th)] = (bits, vals, build_huff(bits, vals, name, tc == 0))
        o += 17 + cnt


def _read_dri(seg, name):
    if len(seg) < 2:
        raise ValueError("%s: bad DRI segment" % name)
    return (seg[0] << 8) | seg[1]


def _markers(d, pos):
    """File offsets and codes of the markers from byte ``pos`` on: 0xFF followed by neither a stuffed zero nor a fill
    byte."""
    ff = np.flatnonzero(d[pos:-1] == 0xFF) + pos
    code = d[ff + 1]
    mk = (code != 0) & (code != 0xFF)
    return ff[mk], code[mk]


def _segments(markers, pos, n, units, ri):
    """The entropy-coded segments of a scan whose data starts at byte ``pos`` of an ``n``-byte file: RST markers up to
    the first other marker (or the end of a truncated file), ``units`` MCUs at ``ri`` per segment (0: one segment).
    Returns ``(segments, end, reason)``: the (start, end) file offsets as an (nseg, 2) int64 array, the offset of the
    marker that ends the scan (``n`` when none does), and why the markers do not fit the interval (else "")."""
    mpos, mcode = markers
    i = int(np.searchsorted(mpos, pos))
    stop = np.flatnonzero((mcode[i:] & 0xF8) != 0xD0)
    j = i + int(stop[0]) if len(stop) else len(mpos)
    end = int(mpos[j]) if j < len(mpos) else n
    ff, nxt = mpos[i:j], mcode[i:j]
    nseg = -(-units // ri) if ri else 1
    if len(ff) > nseg - 1 or (len(ff) and not ri):
        return None, end, "restart markers do not match the restart interval"
    if not np.array_equal(nxt & 7, np.arange(len(ff)) % 8):
        return None, end, "restart markers out of sequence"
    segs = np.full((nseg, 2), end, np.int64)               # segments past a cut have no data (the device flags them)
    segs[:len(ff) + 1, 0] = np.concatenate([[pos], ff + 2])
    segs[:len(ff) + 1, 1] = np.concatenate([ff, [end]])
    return segs, end, ""


def parse(data, name="image"):
    """Headers of one file (bytes or a uint8 array).  Returns a ``JpegInfo``; raises ``ValueError`` naming ``name``
    when the file is not a JPEG the parser can read (truncated or garbled headers)."""
    d = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
    n = len(d)
    info = JpegInfo()
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise ValueError("%s: not a JPEG file (no SOI marker)" % name)
    qt, huff = {}, {}
    jfif = False
    adobe = None
    sof = None
    pos = 2
    while True:
        while pos < n and d[pos] == 0xFF and pos + 1 < n and d[pos + 1] == 0xFF:
            pos += 1                                               # fill bytes
        if pos + 4 > n or d[pos] != 0xFF:
            raise ValueError("%s: truncated or garbled header at byte %d" % (name, pos))
        m = int(d[pos + 1])
        if m == 0xD8 or m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise ValueError("%s: unexpected marker 0x%02X before the scan" % (name, m))
        ln = (int(d[pos + 2]) << 8) | int(d[pos + 3])
        if ln < 2 or pos + 2 + ln > n:
            raise ValueError("%s: segment 0x%02X of length %d runs past the end of the file" % (name, m, ln))
        seg = d[pos + 4:pos + 2 + ln].tobytes()
        pos += 2 + ln
        if m == 0xE0 and seg[:5] == b"JFIF\x00":
            jfif = True
        elif m == 0xE1 and seg[:6] == b"Exif\x00\x00" and info.orientation == 1:
            info.orientation = _exif_orientation(seg)
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            adobe = seg[11]
        elif m == 0xDB:
            o = 0
            while o < len(seg):
                pq, tq = seg[o] >> 4, seg[o] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or o + 1 + size > len(seg):
                    raise ValueError("%s: bad quantisation table" % name)
                q = np.frombuffer(seg, ">u2" if pq else "u1", 64, o + 1).astype(np.int64)
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = q
                qt[tq] = nat
                o += 1 + size
        elif m == 0xC4:
            _read_dht(seg, huff, name)
        elif m == 0xDD:
            info.restart_interval = _read_dri(seg, name)
        elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            if len(seg) < 6 or len(seg) < 6 + 3 * seg[5]:
                raise ValueError("%s: bad SOF segment" % name)
            sof = (m, seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4],
                   [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(seg[5])])
        elif m == 0xCC:
            info.reason = "arithmetic coding"
            return info
        elif m == 0xDA:
            break
    if sof is None:
        raise ValueError("%s: no SOF segment before the scan" % name)
    kind, prec, h, w, comps = sof
    info.h, info.w = h, w
    if not (1 <= h <= MAX_DIMENSION and 1 <= w <= MAX_DIMENSION):
        raise ValueError("%s: image size %dx%d outside 1..%d" % (name, w, h, MAX_DIMENSION))
    info.oh, info.ow = info.size_after_orientation()
    if kind not in (0xC0, 0xC1, 0xC2):
        info.reason = "SOF%d (not sequential or progressive Huffman)" % (kind - 0xC0)
        return info
    if prec != 8:
        info.reason = "%d-bit precision" % prec
        return info
    nc = len(comps)
    if nc == 3:
        cid = [c[0] for c in comps]
        if jfif:
            ycc = True
        elif adobe is not None:
            ycc = adobe == 1
        else:
            ycc = cid != [82, 71, 66]
        if not ycc:
            info.reason = "RGB or Adobe transform %s" % adobe
            return info
        samp = [(c[1], c[2]) for c in comps]
        if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in ((1, 1), (2, 1), (1, 2), (2, 2)):
            info.reason = "sampling %s" % samp
            return info
        info.hs, info.vs = samp[0]
    elif nc == 1:
        info.hs = info.vs = 1                    # a lone component is one non-interleaved scan of plain blocks
    else:
        info.reason = "%d components" % nc
        return info
    info.ncomp = nc
    if w * h * 3 >= 2 ** 62 or info.workspace_bytes() >= 2 ** 62:
        raise ValueError("%s: image too large" % name)
    if kind == 0xC2:
        if any(c[3] not in qt for c in comps):
            raise ValueError("%s: the scan uses an undefined table" % name)
        scans, tables, why = _progressive_scans(d, pos, seg, info, comps, huff, name)
        if why:
            info.reason = "progressive: " + why
            return info
        info.qt = [qt[c[3]] for c in comps]
        info.progressive, info.tables = scans, tables
        info.reason = "SOF2 (not sequential Huffman)"
        return info
    # the SOS header (seg still holds its payload)
    scomp, ss, se, ah, al = _read_sos(seg, name)
    if len(scomp) != nc or [s[0] for s in scomp] != [c[0] for c in comps]:
        info.reason = "multi-scan sequential file"
        return info
    if ss != 0 or se != 63 or ah or al:
        raise ValueError("%s: bad spectral selection in a sequential scan" % name)
    info.qt, info.dc, info.ac = [], [], []
    for (cid, td, ta), c in zip(scomp, comps):
        if c[3] not in qt or (0, td) not in huff or (1, ta) not in huff:
            raise ValueError("%s: the scan uses an undefined table" % name)
        info.qt.append(qt[c[3]])
        info.dc.append(td)
        info.ac.append(ta)
    info.huff = huff
    mx, my = info.mcu
    info.segments, end, why = _segments(_markers(d, pos), pos, n, mx * my, info.restart_interval)
    if why:
        info.reason = why
        return info
    info.eoi = end + 1 < n and d[end + 1] == 0xD9
    info.eligible = True
    return info


def _read_sos(seg, name):
    """(components as (id, DC table, AC table), Ss, Se, Ah, Al) of an SOS payload."""
    ns = seg[0] if seg else 0
    if len(seg) < 4 + 2 * ns or ns < 1:
        raise ValueError("%s: bad SOS segment" % name)
    scomp = [(seg[1 + 2 * i], seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
    return scomp, seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15


def _progressive_scans(d, pos, seg, info, comps, huff, name):
    """The scans of a progressive file whose first SOS payload is ``seg``, with its entropy data at byte ``pos``, up to
    EOI.  Returns ``(scans, tables, reason)``: the ``JpegScan`` list, the ``HUFF`` tables the scans index, and why the
    device does not take the file ("" when it does)."""
    n = len(d)
    cids = [c[0] for c in comps]
    # per component and zigzag coefficient: Al of the last scan that coded it, -1 before any (libjpeg's coef_bits)
    coded = np.full((len(comps), 64), -1, np.int64)
    markers = _markers(d, pos)
    ri = info.restart_interval
    scans, used, index = [], [], {}

    def table(key):
        if key not in huff:
            raise ValueError("%s: the scan uses an undefined table" % name)
        t = huff[key]                            # the table current at this SOS; a later DHT replaces the entry
        if id(t) not in index:
            index[id(t)] = len(used)
            used.append(t)
        return index[id(t)]

    while True:
        if len(scans) == MAX_SCANS:
            return None, None, "more than %d scans" % MAX_SCANS
        k = len(scans)
        scomp, ss, se, ah, al = _read_sos(seg, name)
        idx = [cids.index(s[0]) if s[0] in cids else -1 for s in scomp]
        if -1 in idx or idx != sorted(set(idx)):
            return None, None, "scan %d: components %s not a subset of the frame's in frame order" % (k, idx)
        dc = ss == 0
        # T.81 G.1.1.1, as libjpeg-turbo's jdphuff.c checks it (it refuses the file otherwise)
        if (se != 0 if dc else (se > 63 or ss > se or len(idx) != 1)) or (ah and ah != al + 1) or al > 13:
            return None, None, "scan %d: illegal progression Ss %d Se %d Ah %d Al %d" % (k, ss, se, ah, al)
        # what libjpeg only warns about (a bogus progression) changes its output, so those files stay on the host
        if (coded[idx, ss:se + 1] != (ah if ah else -1)).any() or (not dc and coded[idx[0], 0] < 0):
            return None, None, "scan %d: inconsistent progression Ss %d Se %d Ah %d Al %d" % (k, ss, se, ah, al)
        coded[idx, ss:se + 1] = al
        scan = JpegScan(idx, ss, se, ah, al, [table((0, s[1])) if dc and not ah else 0 for s in scomp],
                        [0 if dc else table((1, s[2])) for s in scomp], ri, None)
        scan.segments, end, why = _segments(markers, pos, n, scan.units(info), ri)
        if why:
            return None, None, "scan %d: %s" % (k, why)
        scans.append(scan)
        if end >= n:
            info.eoi = False                     # cut inside this scan's data, or no EOI after it: the device flags it
            break
        # the markers up to the next scan: tables and restart intervals may change, nothing else may
        pos, m = end, 0
        while m != 0xDA:
            while pos + 1 < n and d[pos] == 0xFF and d[pos + 1] == 0xFF:
                pos += 1                                           # fill bytes
            if pos + 2 > n:
                return None, None, "the file ends between scans"
            if d[pos] != 0xFF:
                return None, None, "extraneous bytes between scans"
            m = int(d[pos + 1])
            if m == 0xD9:
                break
            ln = (int(d[pos + 2]) << 8) | int(d[pos + 3]) if pos + 4 <= n else 0
            if ln < 2 or pos + 2 + ln > n:
                return None, None, "the file ends between scans"
            seg = d[pos + 4:pos + 2 + ln].tobytes()
            pos += 2 + ln
            if m == 0xC4:
                _read_dht(seg, huff, name)
            elif m == 0xDD:
                ri = _read_dri(seg, name)
            elif m != 0xDA and not (0xE0 <= m <= 0xEF or m == 0xFE):
                return None, None, "marker 0x%02X between scans" % m
        if m == 0xD9:
            break
    if (coded != 0).any():
        return None, None, "incomplete progression (libjpeg would smooth the blocks)"
    return scans, [t[2] for t in used], ""


def pack(infos, datas, dst_offsets, alloc=lambda n: np.empty(n, np.uint8)):
    """One ``cpb200_jpeg_decode_batch`` launch over ``infos`` (each ``eligible`` or ``progressive``) with file bytes
    ``datas``: a buffer ``[table (B x 480 B) | per image: Huffman tables | scans (progressive) | segments | file bytes]``
    whose offsets are relative to its own start, so the same device copy is both ``src`` and ``table``.
    ``dst_offsets`` are the byte offsets of the decoded images in ``dst``.  ``alloc(nbytes)`` returns the uint8 host
    buffer.  Returns ``(buffer, workspace_bytes)``."""
    B = len(infos)
    table = np.zeros(B, JPEG_IMAGE)
    up = lambda x, a: x + (-x) % a
    pos = up(table.nbytes, 16)
    ws = 0
    place = []
    for n, (info, data) in enumerate(zip(infos, datas)):
        e = table[n]
        e["huff_offset"] = pos
        if info.progressive is None:
            keys = sorted({(0, t) for t in info.dc} | {(1, t) for t in info.ac})
            tables, segs = [info.huff[k][2] for k in keys], [info.segments]
            for c in range(info.ncomp):
                e["dc_tbl"][c] = keys.index((0, info.dc[c]))
                e["ac_tbl"][c] = keys.index((1, info.ac[c]))
            e["restart_interval"], e["nseg"] = info.restart_interval, len(info.segments)
        else:
            tables, segs = info.tables, [sc.segments for sc in info.progressive]
        pos += len(tables) * HUFF.itemsize
        scans = np.zeros(len(info.progressive or ()), SCAN)
        e["scan_offset"], e["nscan"] = pos, len(scans)
        pos += scans.nbytes
        e["seg_offset"] = pos
        for sc, rec, sg in zip(info.progressive or (), scans, segs):
            rec["seg_offset"], rec["nseg"], rec["restart_interval"] = pos, len(sg), sc.restart_interval
            rec["ncomp"], rec["ss"], rec["se"], rec["ah"], rec["al"] = len(sc.comps), sc.ss, sc.se, sc.ah, sc.al
            rec["comp"][:len(sc.comps)], rec["dc_tbl"][:len(sc.comps)], rec["ac_tbl"][:len(sc.comps)] = \
                sc.comps, sc.dc, sc.ac
            pos += len(sg) * 16
        pos = up(e["seg_offset"] + sum(len(sg) for sg in segs) * 16, 16)
        place.append((tables, scans, segs, pos))
        pos = up(pos + len(data), 16)
        e["coef_offset"] = ws
        nblk = sum(bw * bh for bw, bh in info.blocks())
        e["plane_offset"] = ws + nblk * 128
        ws += nblk * 192
        e["dst_offset"] = dst_offsets[n]
        e["h"], e["w"], e["ncomp"], e["hs"], e["vs"] = info.h, info.w, info.ncomp, info.hs, info.vs
        e["orientation"] = info.orientation
        e["missing_eoi"] = not info.eoi
        for c in range(info.ncomp):
            e["qt"][c] = info.qt[c]
    if pos >= 2 ** 62:
        raise ValueError("jpeg: launch buffer too large")
    buf = alloc(pos)
    hv = buf.numpy() if hasattr(buf, "numpy") else buf
    hv[:table.nbytes] = table.view(np.uint8)
    for data, e, (tables, scans, segs, base) in zip(datas, table, place):
        h0 = int(e["huff_offset"])
        for k, t in enumerate(tables):
            hv[h0 + k * HUFF.itemsize:h0 + (k + 1) * HUFF.itemsize] = t.reshape(1).view(np.uint8)
        s0 = int(e["scan_offset"])
        hv[s0:s0 + scans.nbytes] = scans.view(np.uint8)
        # the parser's segment bounds are file offsets; the kernels read them as offsets into the buffer
        s0 = int(e["seg_offset"])
        sg = np.concatenate(segs) + base
        hv[s0:s0 + sg.nbytes] = sg.astype("<i8").view(np.uint8).reshape(-1)
        hv[base:base + len(data)] = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
    return buf, ws
