"""Host side of the device PNG decoder (``cpb200_png_decode_batch``, ``csrc/png.cu``).

``parse(data, name)`` walks a file's chunks, checks every CRC and decides whether the device can decode it byte for
byte as ``cv2.imread(path, IMREAD_COLOR)`` does (libpng through OpenCV 4.13: 16-bit samples keep their high byte,
1/2/4-bit grayscale is scaled to 8 bits, palettes are expanded with missing entries black, grayscale is replicated to
three channels, alpha is dropped without compositing, ``tRNS`` / ``gAMA`` / ``sBIT`` / ``iCCP`` / ``bKGD`` change
nothing, then OpenCV applies the ``eXIf`` orientation).  ``pack(...)`` lays out the device table of a launch.

The device takes bit depths 1/2/4/8/16 in colour types 0/2/3/4/6, interlaced (Adam7) or not.  What stays with
``cv2.imread`` has ``eligible == False`` and a ``reason``:

- APNG files (an ``acTL`` chunk): ``cv2.imread`` returns the first animation frame, which need not be the ``IDAT``
  image;
- images wider or taller than libpng's default limit (1,000,000) or above OpenCV's 2^30 pixels, which ``cv2.imread``
  refuses.

The kernels trust the table, so every size and offset read from the file is checked here; a file the parser cannot
read (bad signature or CRC, truncated, a bad or oversize IHDR, an unknown critical chunk, IDAT chunks that are not
consecutive, a missing or duplicate palette) raises ``ValueError`` naming the image.  ``cv2.imread`` refuses those files too.
"""
from __future__ import annotations

import zlib

import numpy as np

from .jpeg import oriented_size, tiff_orientation

SIGNATURE = b"\x89PNG\r\n\x1a\n"
# the C ABI entry point that decodes a launch packed by pack()
KERNEL = "png_decode_batch"
# bit depths libpng accepts per colour type (PNG spec 11.2.2)
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# libpng's default user limit on width and height, and OpenCV's limit on the pixels of a decoded image
MAX_DIMENSION = 1000000
MAX_PIXELS = 1 << 30
# Adam7: (x start, y start, x step, y step) of passes 1..7
ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2))
# bytes after each zlib stream in the launch buffer: the bit reader loads 8-byte words up to 24 bytes past its end
STREAM_PAD = 32

# struct cpb200_png_image (include/centerpose_b200.h)
PNG_IMAGE = np.dtype([("src_offset", "<i8"), ("src_bytes", "<i8"), ("palette_offset", "<i8"), ("ws_offset", "<i8"),
                      ("ws_bytes", "<i8"), ("dst_offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("color_type", "<i4"),
                      ("depth", "<i4"), ("interlace", "<i4"), ("orientation", "<i4")])
assert PNG_IMAGE.itemsize == 72


class PngInfo:
    """What ``parse`` found.  ``eligible`` says whether the device decodes the file (``reason`` says why not).  ``h, w``
    the stored size, ``oh, ow`` the size after the EXIF ``orientation`` (what ``cv2.imread`` returns), ``color_type``,
    ``depth``, ``interlace``, ``palette`` (the PLTE payload, RGB triples, or None) and ``idat``, the (start, end) file
    offsets of the IDAT payloads, whose concatenation is the zlib stream."""

    def __init__(self):
        self.eligible = False
        self.reason = ""
        self.orientation = 1
        self.palette = None
        self.idat = []

    def passes(self):
        """(width, height) of each non-empty reduced image: the seven Adam7 passes, or the whole image."""
        if not self.interlace:
            return [(self.w, self.h)]
        out = []
        for x0, y0, dx, dy in ADAM7:
            pw, ph = -(-(self.w - x0) // dx), -(-(self.h - y0) // dy)
            if pw > 0 and ph > 0:
                out.append((pw, ph))
        return out

    def row_bytes(self, pw):
        return -(-pw * CHANNELS[self.color_type] * self.depth // 8)

    def filtered_bytes(self):
        """Size of the inflated stream: per pass, rows of one filter-type byte and the packed samples."""
        return sum(ph * (1 + self.row_bytes(pw)) for pw, ph in self.passes())

    def workspace_bytes(self):
        """The filtered scanlines (unfiltered in place) rounded up to 16 bytes, then 16 bytes for the Adler-32 the
        inflate kernel reads from the stream."""
        return -(-self.filtered_bytes() // 16) * 16 + 16

    def stream_bytes(self):
        return sum(b - a for a, b in self.idat)


def parse(data, name="image"):
    """Chunks of one file (bytes or a uint8 array).  Returns a ``PngInfo``; raises ``ValueError`` naming ``name`` when
    the file is not a PNG the parser can read."""
    d = data.tobytes() if isinstance(data, np.ndarray) else bytes(data)
    n = len(d)
    if d[:8] != SIGNATURE:
        raise ValueError("%s: not a PNG file (no signature)" % name)
    info = PngInfo()
    pos, ihdr, end, last = 8, None, False, None
    apng = exif = plte = False
    while not end:
        if pos + 12 > n:
            raise ValueError("%s: truncated at byte %d (no IEND chunk)" % (name, pos))
        ln = int.from_bytes(d[pos:pos + 4], "big")
        ctype = d[pos + 4:pos + 8]
        if ln > 0x7FFFFFFF or pos + 12 + ln > n:
            raise ValueError("%s: chunk %r of length %d runs past the end of the file" % (name, ctype, ln))
        body = d[pos + 8:pos + 8 + ln]
        if zlib.crc32(ctype + body) != int.from_bytes(d[pos + 8 + ln:pos + 12 + ln], "big"):
            raise ValueError("%s: CRC error in chunk %r" % (name, ctype))
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in ctype):
            raise ValueError("%s: bad chunk type %r" % (name, ctype))
        if ihdr is None and ctype != b"IHDR":
            raise ValueError("%s: the first chunk is %r, not IHDR" % (name, ctype))
        if ctype == b"IHDR":
            if ihdr is not None or ln != 13:
                raise ValueError("%s: bad IHDR chunk" % name)
            ihdr = body
            w, h = int.from_bytes(body[0:4], "big"), int.from_bytes(body[4:8], "big")
            depth, ct, comp, filt, inter = body[8:13]
            if not (1 <= w <= 0x7FFFFFFF and 1 <= h <= 0x7FFFFFFF):
                raise ValueError("%s: image size %dx%d outside 1..2^31-1" % (name, w, h))
            if ct not in DEPTHS or depth not in DEPTHS[ct] or comp or filt or inter > 1:
                raise ValueError("%s: bad IHDR (colour type %d, depth %d, methods %d/%d/%d)"
                                 % (name, ct, depth, comp, filt, inter))
            info.h, info.w, info.depth, info.color_type, info.interlace = h, w, depth, ct, inter
        elif ctype == b"PLTE":
            if ln == 0 or ln % 3 or ln > 3 * 256 or info.idat or plte:
                raise ValueError("%s: bad or duplicate PLTE chunk" % name)   # libpng stops at a second PLTE
            plte = True
            if ct == 0 or ct == 4:
                raise ValueError("%s: PLTE in a grayscale image" % name)
            info.palette = body
        elif ctype == b"IDAT":
            if info.idat and last != b"IDAT":
                raise ValueError("%s: IDAT chunks are not consecutive" % name)
            info.idat.append((pos + 8, pos + 8 + ln))
        elif ctype == b"IEND":
            end = True
        elif ctype == b"eXIf":
            if not exif:                                  # libpng keeps the first eXIf chunk
                exif = True
                info.orientation = tiff_orientation(body)
        elif ctype == b"acTL":
            apng = True
        elif ctype[0] < 97:
            raise ValueError("%s: unknown critical chunk %r" % (name, ctype))
        last = ctype
        pos += 12 + ln
    if not info.idat:
        raise ValueError("%s: no IDAT chunk" % name)
    if ct == 3 and info.palette is None:
        raise ValueError("%s: palette image without PLTE" % name)
    if ct != 3:
        info.palette = None                           # a suggested palette of a truecolour image changes nothing
    info.oh, info.ow = oriented_size(info.h, info.w, info.orientation)
    if apng:
        info.reason = "APNG (cv2.imread returns the first animation frame)"
    elif w > MAX_DIMENSION or h > MAX_DIMENSION or w * h > MAX_PIXELS:
        info.reason = "image size %dx%d above what cv2.imread reads" % (w, h)
    else:
        info.eligible = True
    return info


def pack(infos, datas, dst_offsets, alloc=lambda n: np.empty(n, np.uint8)):
    """One ``cpb200_png_decode_batch`` launch over the ``eligible`` ``infos`` with file bytes ``datas``: a buffer
    ``[table (B x 72 B) | per image: zlib stream (the IDAT payloads back to back) + 32 bytes | palette (768 B, entries
    past PLTE black)]``, each part 16-byte aligned, whose offsets are relative to its own start, so the same device copy
    is both ``src`` and ``table``.  ``dst_offsets`` are the byte offsets of the decoded images in ``dst``.
    ``alloc(nbytes)`` returns the uint8 host buffer.  Returns ``(buffer, workspace_bytes)``."""
    B = len(infos)
    table = np.zeros(B, PNG_IMAGE)
    up = lambda x, a: x + (-x) % a
    pos, ws = up(table.nbytes, 16), 0
    for n, info in enumerate(infos):
        if not info.eligible:
            raise ValueError("png.pack: image %d is not eligible (%s)" % (n, info.reason))
        e = table[n]
        e["src_offset"], e["src_bytes"] = pos, info.stream_bytes()
        pos = up(pos + info.stream_bytes() + STREAM_PAD, 16)
        if info.palette is not None:
            e["palette_offset"] = pos
            pos += 768
        e["ws_offset"], e["ws_bytes"] = ws, info.workspace_bytes()
        ws += info.workspace_bytes()
        e["dst_offset"] = dst_offsets[n]
        e["h"], e["w"], e["color_type"], e["depth"] = info.h, info.w, info.color_type, info.depth
        e["interlace"], e["orientation"] = info.interlace, info.orientation
    if pos >= 2 ** 62 or ws >= 2 ** 62:
        raise ValueError("png: launch buffer too large")
    buf = alloc(pos)
    hv = buf.numpy() if hasattr(buf, "numpy") else buf
    hv[:table.nbytes] = table.view(np.uint8)
    for info, data, e in zip(infos, datas, table):
        d = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
        o = int(e["src_offset"])
        for a, b in info.idat:
            hv[o:o + b - a] = d[a:b]
            o += b - a
        hv[o:o + STREAM_PAD] = 0
        if info.palette is not None:
            p = int(e["palette_offset"])
            hv[p:p + 768] = 0
            hv[p:p + len(info.palette)] = np.frombuffer(info.palette, np.uint8)
    return buf, ws
