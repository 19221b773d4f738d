"""Host side of the device lossless WebP decoder (``cpb200_webp_lossless_decode_batch``, ``csrc/webp_lossless.cu``).

``parse(data, name)`` walks a file's RIFF chunks (``webp.walk``) and reads the 5-byte VP8L header (signature 0x2f,
14-bit width - 1 and height - 1, the alpha hint, 3 version bits), and decides whether the device can decode it byte
for byte as ``cv2.imread(path, IMREAD_COLOR)`` does (libwebp through OpenCV 4.13: the ARGB image with its alpha
dropped, then OpenCV applies the orientation of the first ``EXIF`` chunk when the ``VP8X`` header flags one).  It
decodes no entropy-coded data, so a file costs a few microseconds here.  ``pack(...)`` lays out the device table of a
launch.

The device takes a ``VP8L`` image in the simple container, or in the extended one (``VP8X``) with ``ICCP``, ``XMP ``,
``EXIF`` and unknown chunks around it.  This is what ``cv2.imwrite`` / ``cv2.imencode`` write for ``.webp`` with no
parameters or a quality above 100.  What stays with ``cv2.imread`` has ``eligible == False`` and a ``reason``:
animated files, and a RIFF size other than the file's size less 8.

A file the parser cannot read (what ``webp.walk`` refuses, a file under 32 bytes, no ``VP8L`` chunk, a chunk shorter
than the header, a signature byte other than 0x2f, a version other than 0, a ``VP8X`` canvas other than the image's
size) raises ``ValueError`` naming the image; ``cv2.imread`` refuses those files too.  Whether the entropy-coded stream is valid is
found on the device (status 1).

The number of prefix-code groups sits inside the entropy-coded stream, so the workspace holds a fixed budget of
``MAX_GROUPS`` groups; a file that needs more gets status 2 on the device and is read by ``cv2.imread``.
"""
from __future__ import annotations

import numpy as np

from .jpeg import oriented_size
from .webp import STREAM_PAD, walk

# the C ABI entry point that decodes a launch packed by pack()
KERNEL = "webp_lossless_decode_batch"
# prefix-code groups per image on the device (CPB200_WEBP_LOSSLESS_MAX_GROUPS).  cv2.imencode's default files use at
# most 37 over the 256 benchmark files of tools/bench_webp.py --lossless, which prints the count
MAX_GROUPS = 64
# workspace of one group: five codes of a 256-entry lookup table and 16 counts (uint16), and the sorted symbols of
# the green (280 + 2048 cache entries), red, blue, alpha and distance (40) alphabets
GROUP_BYTES = 5 * 256 * 2 + 5 * 16 * 2 + (280 + 2048 + 3 * 256 + 40) * 2
HEADER_BYTES = 128
# cv2.imread refuses a WebP file shorter than this
MIN_FILE_BYTES = 32

# struct cpb200_webp_lossless_image (include/centerpose_b200.h)
WEBP_LOSSLESS_IMAGE = np.dtype([("src_offset", "<i8"), ("src_bytes", "<i8"), ("ws_offset", "<i8"),
                                ("ws_bytes", "<i8"), ("dst_offset", "<i8"), ("h", "<i4"), ("w", "<i4"),
                                ("orientation", "<i4"), ("pad", "<i4")])
assert WEBP_LOSSLESS_IMAGE.itemsize == 56


def workspace_bytes(w, h):
    """Device workspace of a w x h image: a 128-byte header, two ARGB planes (the coded image and the output of
    colour indexing), the sub-images (predictor, cross-colour and entropy images of at most ceil(w/4) x ceil(h/4)
    pixels each, the 256-entry palette) and ``MAX_GROUPS`` prefix-code groups (csrc/webp_lossless.cu ``layout``)."""
    up = lambda x: x + (-x) % 16
    tiles = ((w + 3) >> 2) * ((h + 3) >> 2)
    return HEADER_BYTES + 2 * up(4 * w * h) + up(4 * (3 * tiles + 256)) + MAX_GROUPS * GROUP_BYTES


class WebpLosslessInfo:
    """What ``parse`` found.  ``eligible`` says whether the device decodes the file (``reason`` says why not).  ``h,
    w`` the image size, ``oh, ow`` the size after the EXIF ``orientation`` (what ``cv2.imread`` returns), ``vp8l`` the
    file offset of the VP8L payload.  The decoder reads from there to the end of the file, as libwebp reads to the
    end of the data it was given."""

    def __init__(self):
        self.eligible = False
        self.reason = ""
        self.orientation = 1
        self.vp8l = None
        self.size = 0

    def workspace_bytes(self):
        return workspace_bytes(self.w, self.h)

    def stream_bytes(self):
        return self.size - self.vp8l


def parse(data, name="image"):
    """Chunks and VP8L header of one file (bytes or a uint8 array).  Returns a ``WebpLosslessInfo``; raises
    ``ValueError`` naming ``name`` when the file is not a lossless WebP file the parser can read."""
    d = data.tobytes() if isinstance(data, np.ndarray) else bytes(data)
    c = walk(d, name)
    if len(d) < MIN_FILE_BYTES:
        raise ValueError("%s: %d bytes, shorter than the %d cv2.imread reads" % (name, len(d), MIN_FILE_BYTES))
    info = WebpLosslessInfo()
    info.size = len(d)
    if c.animated():
        info.reason = "animated WebP"
        return info
    if c.image != b"VP8L":
        raise ValueError("%s: no VP8L image chunk" % name)
    if c.length < 5:
        raise ValueError("%s: VP8L chunk of %d bytes is shorter than its header" % (name, c.length))
    hdr = d[c.body:c.body + 5]
    if hdr[0] != 0x2F:
        raise ValueError("%s: bad VP8L signature 0x%02x" % (name, hdr[0]))
    if hdr[4] >> 5:
        raise ValueError("%s: VP8L version %d" % (name, hdr[4] >> 5))
    v = int.from_bytes(hdr[1:5], "little")
    info.w, info.h = (v & 0x3FFF) + 1, ((v >> 14) & 0x3FFF) + 1
    if c.canvas is not None and c.canvas != (info.w, info.h):
        raise ValueError("%s: VP8X canvas %dx%d differs from the %dx%d image" % (name, *c.canvas, info.w, info.h))
    info.vp8l = c.body
    info.orientation = c.orientation()
    info.oh, info.ow = oriented_size(info.h, info.w, info.orientation)
    if c.riff + 8 != info.size:
        info.reason = "RIFF size %d disagrees with the file's %d bytes" % (c.riff, info.size)
    else:
        info.eligible = True
    return info


def pack(infos, datas, dst_offsets, alloc=lambda n: np.empty(n, np.uint8)):
    """One ``cpb200_webp_lossless_decode_batch`` launch over the ``eligible`` ``infos`` with file bytes ``datas``: a
    buffer ``[table (B x 56 B) | per image: the file from its VP8L payload to its end + 32 zero bytes]``, each part
    16-byte aligned, whose offsets are relative to its own start, so the same device copy is both ``src`` and
    ``table``.  ``dst_offsets`` are the byte offsets of the decoded images in ``dst``.  ``alloc(nbytes)`` returns the
    uint8 host buffer.  Returns ``(buffer, workspace_bytes)``."""
    B = len(infos)
    table = np.zeros(B, WEBP_LOSSLESS_IMAGE)
    up = lambda x, a: x + (-x) % a
    pos, ws = up(table.nbytes, 16), 0
    for k, info in enumerate(infos):
        if not info.eligible:
            raise ValueError("webp_lossless.pack: image %d is not eligible (%s)" % (k, info.reason))
        e = table[k]
        e["src_offset"], e["src_bytes"] = pos, info.stream_bytes()
        pos = up(pos + info.stream_bytes() + STREAM_PAD, 16)
        e["ws_offset"], e["ws_bytes"] = ws, info.workspace_bytes()
        ws += info.workspace_bytes()
        e["dst_offset"] = dst_offsets[k]
        e["h"], e["w"], e["orientation"] = info.h, info.w, info.orientation
    if pos >= 2 ** 62 or ws >= 2 ** 62:
        raise ValueError("webp_lossless: launch buffer too large")
    buf = alloc(pos)
    hv = buf.numpy() if hasattr(buf, "numpy") else buf
    hv[:table.nbytes] = table.view(np.uint8)
    for info, data, e in zip(infos, datas, table):
        d = np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data
        o, nb = int(e["src_offset"]), info.stream_bytes()
        hv[o:o + nb] = d[info.vp8l:info.vp8l + nb]
        hv[o + nb:o + nb + STREAM_PAD] = 0
    return buf, ws
