"""Host side of the device WebP decoder (``cpb200_webp_decode_batch``, ``csrc/webp.cu``).

``parse(data, name)`` walks a file's RIFF chunks and reads the 10-byte uncompressed header of its VP8 key frame (frame
tag, start code, size), and decides whether the device can decode it byte for byte as ``cv2.imread(path,
IMREAD_COLOR)`` does (libwebp through OpenCV 4.13: fancy 4:2:0 upsampling, libwebp's fixed-point YUV -> BGR, then
OpenCV applies the orientation of the first ``EXIF`` chunk when the ``VP8X`` header flags one).  It decodes no
bool-coded data, so a file costs a few microseconds here.  ``pack(...)`` lays out the device table of a launch.

The device takes lossy files: a ``VP8 `` image in the simple container, or in the extended one (``VP8X``) with
``ICCP``, ``XMP ``, ``EXIF`` and unknown chunks around it, which change no pixel.  What stays with ``cv2.imread``
has ``eligible == False`` and a ``reason``:

- lossless files (``VP8L``);
- files with an alpha channel (``ALPH``);
- animated files (``ANIM`` / ``ANMF``, or the animation flag);
- a RIFF size other than the file's size less 8 (cv2.imread ignores bytes past the RIFF chunk and refuses a file
  shorter than it).

A file the parser cannot read (no RIFF / WEBP signature, a chunk past the end, a first chunk other than ``VP8X``,
``VP8 `` or ``VP8L``, no image chunk, a ``VP8X`` canvas other
than the frame's size, a frame tag that is not a shown key frame of profile 0..3, a bad start code, a first partition
longer than the chunk, a zero width or height) raises ``ValueError`` naming the image.  ``cv2.imread`` refuses those
files too.  Whether the bool-coded partitions hold enough data is found on the device (status 1).
"""
from __future__ import annotations

import struct

import numpy as np

from .jpeg import oriented_size, tiff_orientation

SIGNATURE = b"RIFF"
FORMAT = b"WEBP"
# the C ABI entry point that decodes a launch packed by pack()
KERNEL = "webp_decode_batch"
# bytes after each VP8 payload in the launch buffer: the bool decoder reads 8 bytes at a time
STREAM_PAD = 32
# workspace per 16x16 macroblock: modes and filter strength (32 B), int16 coefficients (768 B), Y / U / V planes
# (256 + 64 + 64 B); plus 16 bytes of frame flags per image
MB_WORKSPACE = 32 + 768 + 256 + 128
# VP8X flags
VP8X_ANIMATION, VP8X_EXIF = 0x02, 0x08

# struct cpb200_webp_image (include/centerpose_b200.h)
WEBP_IMAGE = np.dtype([("src_offset", "<i8"), ("src_bytes", "<i8"), ("ws_offset", "<i8"), ("ws_bytes", "<i8"),
                       ("dst_offset", "<i8"), ("h", "<i4"), ("w", "<i4"), ("orientation", "<i4"), ("pad", "<i4")])
assert WEBP_IMAGE.itemsize == 56


def is_webp(data):
    """True when ``data`` starts like a WebP file (``RIFF`` .... ``WEBP``)."""
    return bytes(data[:4]) == SIGNATURE and bytes(data[8:12]) == FORMAT


class WebpInfo:
    """What ``parse`` found.  ``eligible`` says whether the device decodes the file (``reason`` says why not).  ``h,
    w`` the frame size, ``oh, ow`` the size after the EXIF ``orientation`` (what ``cv2.imread`` returns), ``vp8``
    the file offset of the VP8 payload (the frame tag).  The decoder reads from there to the end of the file, as
    libwebp does: its last partition runs to the end of the data it was given."""

    def __init__(self):
        self.eligible = False
        self.reason = ""
        self.orientation = 1
        self.vp8 = None
        self.size = 0

    def macroblocks(self):
        return ((self.w + 15) >> 4) * ((self.h + 15) >> 4)

    def workspace_bytes(self):
        return 16 + MB_WORKSPACE * self.macroblocks()

    def stream_bytes(self):
        return self.size - self.vp8


def _frame_header(d, pos, ln, name):
    """(first partition size, width, height) of the VP8 key frame whose payload starts at ``pos`` (RFC 6386 9.1)."""
    if ln < 10:
        raise ValueError("%s: VP8 chunk of %d bytes is shorter than its frame header" % (name, ln))
    tag = d[pos] | d[pos + 1] << 8 | d[pos + 2] << 16
    if tag & 1:
        raise ValueError("%s: the VP8 frame is not a key frame" % name)
    if (tag >> 1) & 7 > 3 or not (tag >> 4) & 1:
        raise ValueError("%s: bad VP8 frame tag (profile %d, show %d)" % (name, (tag >> 1) & 7, (tag >> 4) & 1))
    if d[pos + 3:pos + 6] != b"\x9d\x01\x2a":
        raise ValueError("%s: bad VP8 start code" % name)
    part0 = tag >> 5
    w, h = struct.unpack_from("<HH", d, pos + 6)
    w, h = w & 0x3FFF, h & 0x3FFF                     # the upscaling bits are ignored, as libwebp does
    if not w or not h:
        raise ValueError("%s: VP8 frame of size %dx%d" % (name, w, h))
    if part0 > ln - 10:
        raise ValueError("%s: first partition of %d bytes runs past the VP8 chunk" % (name, part0))
    return part0, w, h


class Chunks:
    """What ``walk`` found in a file's RIFF chunk list: ``riff`` its RIFF size, ``flags`` and ``canvas`` (w, h) of the
    ``VP8X`` chunk (``canvas`` None in the simple container), ``image`` the FourCC of the first ``VP8 `` / ``VP8L``
    chunk with its payload offset ``body`` and length ``length``, ``exif`` the first ``EXIF`` payload, and whether a
    ``VP8L`` (``lossless``), ``ALPH`` (``alpha``) or ``ANIM`` / ``ANMF`` (``anim``) chunk was seen.  ``tail_error`` says
    why the walk stopped at a bad chunk after the image chunk, which libwebp never reads."""

    def __init__(self, riff):
        self.riff, self.flags, self.canvas, self.exif = riff, 0, None, None
        self.image, self.body, self.length = None, None, 0
        self.lossless = self.alpha = self.anim = False
        self.tail_error = None

    def animated(self):
        return self.anim or bool(self.flags & VP8X_ANIMATION)

    def orientation(self):
        """The EXIF orientation cv2.imread applies: only when ``VP8X`` flags EXIF, from a bare TIFF header (an
        "Exif\\0\\0" prefix is ignored), and not when a bad chunk follows the image (cv2.imread then reads the
        image without its metadata)."""
        if self.canvas is not None and self.flags & VP8X_EXIF and self.exif is not None and self.tail_error is None:
            return tiff_orientation(self.exif)
        return 1


def walk(d, name):
    """The chunk list of file bytes ``d`` (the simple container ends at its image chunk, as libwebp reads it).  Raises
    ``ValueError`` naming ``name`` where cv2.imread refuses the container: no RIFF / WEBP signature, a chunk past the
    end or a bad ``VP8X`` chunk before the image chunk, a first chunk other than ``VP8X``, ``VP8 `` or ``VP8L``.  The
    same faults after the image chunk end the walk with ``tail_error`` set."""
    n = len(d)
    if n < 12 or not is_webp(d):
        raise ValueError("%s: not a WebP file (no RIFF / WEBP signature)" % name)
    c = Chunks(struct.unpack_from("<I", d, 4)[0])
    end = min(n, c.riff + 8)
    pos, first = 12, True
    while pos + 8 <= end:
        ctype, ln = d[pos:pos + 4], struct.unpack_from("<I", d, pos + 4)[0]
        body = pos + 8
        err = None
        if body + ln > end:
            err = "%s: chunk %r of %d bytes runs past the end of the file" % (name, ctype, ln)
        elif ctype == b"VP8X" and (not first or ln != 10):
            err = "%s: bad VP8X chunk" % name
        if err is not None:
            if c.image is None:
                raise ValueError(err)
            c.tail_error = err
            break
        if first and ctype not in (b"VP8X", b"VP8 ", b"VP8L"):
            # without VP8X, libwebp reads the first chunk as the image bitstream, and cv2.imread fails
            raise ValueError("%s: first chunk %r is neither VP8X nor an image" % (name, ctype))
        if ctype == b"VP8X":
            c.flags = d[body]
            c.canvas = (1 + int.from_bytes(d[body + 4:body + 7], "little"),
                        1 + int.from_bytes(d[body + 7:body + 10], "little"))
        elif ctype in (b"VP8 ", b"VP8L"):
            c.lossless |= ctype == b"VP8L"
            if c.image is None:
                c.image, c.body, c.length = ctype, body, ln
                if c.canvas is None:                  # the simple container: nothing after the image is read
                    break
        elif ctype == b"ALPH":
            c.alpha = True
        elif ctype in (b"ANIM", b"ANMF"):
            c.anim = True
        elif ctype == b"EXIF":
            if c.exif is None:
                c.exif = d[body:body + ln]            # cv2.imread reads the first EXIF chunk
        first = False
        pos = body + ln + (ln & 1)
    return c


def parse(data, name="image"):
    """Chunks of one file (bytes or a uint8 array).  Returns a ``WebpInfo``; raises ``ValueError`` naming ``name``
    when the file is not a WebP file the parser can read."""
    d = data.tobytes() if isinstance(data, np.ndarray) else bytes(data)
    c = walk(d, name)
    info = WebpInfo()
    info.size = len(d)
    if c.lossless:
        info.reason = "lossless WebP (VP8L)"
        return info
    if c.tail_error:
        raise ValueError(c.tail_error)
    if c.animated():
        info.reason = "animated WebP"
        return info
    if c.image is None:
        raise ValueError("%s: no VP8 image chunk" % name)
    _, info.w, info.h = _frame_header(d, c.body, c.length, name)
    info.vp8 = c.body
    if c.canvas is not None and c.canvas != (info.w, info.h):
        raise ValueError("%s: VP8X canvas %dx%d differs from the %dx%d frame" % (name, *c.canvas, info.w, info.h))
    info.orientation = c.orientation()
    info.oh, info.ow = oriented_size(info.h, info.w, info.orientation)
    if c.alpha:
        info.reason = "WebP with an alpha channel (ALPH)"
    elif c.riff + 8 != info.size:
        info.reason = "RIFF size %d disagrees with the file's %d bytes" % (c.riff, info.size)
    else:
        info.eligible = True
    return info


def pack(infos, datas, dst_offsets, alloc=lambda n: np.empty(n, np.uint8)):
    """One ``cpb200_webp_decode_batch`` launch over the ``eligible`` ``infos`` with file bytes ``datas``: a buffer
    ``[table (B x 56 B) | per image: the file from its VP8 payload to its end + 32 bytes]``, each part 16-byte aligned,
    whose offsets are relative to its own start, so the same device copy is both ``src`` and ``table``.
    ``dst_offsets`` are the byte offsets of the decoded images in ``dst``.  ``alloc(nbytes)`` returns the uint8 host
    buffer.  Returns ``(buffer, workspace_bytes)``."""
    B = len(infos)
    table = np.zeros(B, WEBP_IMAGE)
    up = lambda x, a: x + (-x) % a
    pos, ws = up(table.nbytes, 16), 0
    for k, info in enumerate(infos):
        if not info.eligible:
            raise ValueError("webp.pack: image %d is not eligible (%s)" % (k, info.reason))
        e = table[k]
        e["src_offset"], e["src_bytes"] = pos, info.stream_bytes()
        pos = up(pos + info.stream_bytes() + STREAM_PAD, 16)
        e["ws_offset"], e["ws_bytes"] = ws, info.workspace_bytes()
        ws += info.workspace_bytes()
        e["dst_offset"] = dst_offsets[k]
        e["h"], e["w"], e["orientation"] = info.h, info.w, info.orientation
    if pos >= 2 ** 62 or ws >= 2 ** 62:
        raise ValueError("webp: launch buffer too large")
    buf = alloc(pos)
    hv = buf.numpy() if hasattr(buf, "numpy") else buf
    hv[:table.nbytes] = table.view(np.uint8)
    for info, data, e in zip(infos, datas, table):
        d = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
        o, nb = int(e["src_offset"]), info.stream_bytes()
        hv[o:o + nb] = d[info.vp8:info.vp8 + nb]
        hv[o + nb:o + nb + STREAM_PAD] = 0
    return buf, ws
