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

The other direction, ``cv2.imencode('.png', img)`` byte for byte on the device (``cpb200_png_encode_batch``,
``csrc/png_encode.cu``): ``encode(images)`` returns the files of BGR uint8 host arrays or CUDA tensors, and
``encode_layout`` / ``encode_launch`` encode images already on the device where they are.
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


# ---- encoding: cv2.imencode('.png', img) on the device ----
#
# OpenCV 4.13 writes a BGR uint8 image through libpng with the Sub filter (None on one-pixel rows), zlib level 1,
# strategy Z_RLE and memLevel 8, so the file is fixed by the pixels.  zlib's _tr_flush_block may only store a block
# whose start is still in the window; here it always is when storing could win.  Up to 16 KiB of scanlines the window
# holds all of them (libpng sizes it so, and zlib slides only past 2 * window - 262 bytes).  Past that a block's start
# leaves the 32 KiB window only if the block covers more than 32506 bytes with at most 16383 symbols, and then its
# static coding, which bounds zlib's estimate, costs at most 9 bits per literal and 4 bits per matched byte: under 8
# bits per byte, so storing (8 bits per byte plus 4 bytes) never wins and the rule never decides.

ENCODE_KERNEL = "png_encode_batch"
# struct cpb200_png_encode_image (include/centerpose_b200.h)
ENCODE_IMAGE = np.dtype([("src", "<u8"), ("pitch", "<i8"), ("filt_offset", "<i8"), ("sym_offset", "<i8"),
                         ("tile_offset", "<i8"), ("block_offset", "<i8"), ("state_offset", "<i8"), ("z_offset", "<i8"),
                         ("z_bytes", "<i8"), ("h", "<i4"), ("w", "<i4"), ("tile0", "<i4"), ("block0", "<i4"),
                         ("chunk0", "<i4"), ("pad", "<i4")])
assert ENCODE_IMAGE.itemsize == 96
# CPB200_PNG_ENCODE_TILE / _TILE_REC / _BLOCK_REC / _STATE_REC
ENCODE_TILE, TILE_REC, BLOCK_REC, STATE_REC = 4096, 32, 1088, 64
# zlib's symbol buffer at memLevel 8 (lit_bufsize - 1) and libpng's IDAT size
BLOCK_SYMBOLS = 16383
IDAT_BYTES = 8192


def filtered_size(h, w):
    """Bytes of the scanlines libpng deflates: per row a filter-type byte and 3 * w samples."""
    return h * (1 + 3 * w)


def deflate_bound(n):
    """zlib's deflateBound of n bytes with the zlib wrapper, in the conservative form it uses for parameters other
    than its defaults (libpng lowers windowBits for small images)."""
    return n + ((n + 7) >> 3) + ((n + 63) >> 6) + 5 + 6


def encode_bound(h, w):
    """An upper bound of the PNG file size of an h x w image: signature, IHDR, the bound zlib stream in IDAT chunks,
    IEND."""
    zb = deflate_bound(filtered_size(h, w))
    return 8 + 25 + 12 * -(-zb // IDAT_BYTES) + zb + 12


def encode_layout(sources, shapes, pitches):
    """The launch table of images at device addresses ``sources`` with ``(h, w)`` ``shapes`` and row ``pitches`` in
    bytes.  Returns ``(table, (tiles, blocks, chunks), workspace_bytes, out_bytes)``: the slot counts of the launch,
    the workspace it needs and the output bytes that hold every file (the sum of ``encode_bound``)."""
    table = np.zeros(len(shapes), ENCODE_IMAGE)
    up = lambda x, a: x + (-x) % a
    ws = tiles = blocks = chunks = out = 0
    for e, src, (h, w), pitch in zip(table, sources, shapes, pitches):
        n = filtered_size(h, w)
        if not (h >= 1 and w >= 1 and pitch >= 3 * w and n < 2 ** 31):
            raise ValueError("png.encode: a %dx%d image with row pitch %d cannot be encoded" % (h, w, pitch))
        e["src"], e["pitch"], e["h"], e["w"] = src, pitch, h, w
        nt, nb = -(-n // ENCODE_TILE), n // BLOCK_SYMBOLS + 1
        e["filt_offset"] = ws
        e["sym_offset"] = ws = up(ws + n, 16)
        e["tile_offset"] = ws = up(ws + 2 * n, 16)
        e["block_offset"] = ws = ws + nt * TILE_REC
        e["state_offset"] = ws = ws + nb * BLOCK_REC
        e["z_offset"] = ws = up(ws + STATE_REC, 16)
        e["z_bytes"] = up(deflate_bound(n) + 8, 16)
        ws += int(e["z_bytes"])
        e["tile0"], e["block0"], e["chunk0"] = tiles, blocks, chunks
        tiles, blocks, chunks = tiles + nt, blocks + nb, chunks + -(-int(e["z_bytes"]) // IDAT_BYTES)
        out += encode_bound(h, w)
    if len(table) > 65535 or chunks >= 2 ** 31:
        raise ValueError("png.encode: %d images exceed one launch" % len(table))
    return table, (tiles, blocks, chunks), max(ws, 16), max(out, 1)


def encode_launch(table, counts, workspace_bytes, out, sizes):
    """One upload of ``table`` and one ``cpb200_png_encode_batch`` on the current stream: the files back to back from
    byte 0 of the uint8 CUDA tensor ``out``, their sizes into the int64 CUDA tensor ``sizes``."""
    import torch
    from . import _lib
    dev = out.device
    host = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).pin_memory()
    buf = host.to(dev, non_blocking=True)
    ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = _lib.lib().cpb200_png_encode_batch(buf.data_ptr(), len(table), *counts, ws.data_ptr(), out.data_ptr(),
                                                sizes.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(st, ENCODE_KERNEL)


def download_files(out, sizes):
    """One read of the sizes and one copy of the packed files: one ``bytes`` per image."""
    sz = sizes.cpu().numpy()
    ends = np.cumsum(sz)
    data = out[:int(ends[-1])].cpu().numpy().tobytes()
    return [data[e - s:e] for s, e in zip(sz.tolist(), ends.tolist())]


def encode(images):
    """``cv2.imencode('.png', img)[1].tobytes()`` of each BGR uint8 ``(H, W, 3)`` image, a host array or a CUDA tensor,
    on the device: one upload of the host arrays, one launch, one read of the sizes and one copy of the files.  A CUDA
    tensor is read where it is when its pixels are packed (strides (pitch, 3, 1)).  Anything else raises
    ``ValueError`` before any launch."""
    import torch
    images = list(images)
    dev = None
    for i, im in enumerate(images):
        if isinstance(im, torch.Tensor):
            if not im.is_cuda:
                raise ValueError("png.encode: image %d is a CPU tensor; pass a numpy array or a CUDA tensor" % i)
            dev = dev or im.device
            if im.device != dev:
                raise ValueError("png.encode: image %d is on %s, image 0 on %s" % (i, im.device, dev))
            dtype, shape = im.dtype, tuple(im.shape)
            ok = dtype == torch.uint8
        elif isinstance(im, np.ndarray):
            dtype, shape = im.dtype, im.shape
            ok = dtype == np.uint8
        else:
            raise ValueError("png.encode: image %d is a %s, not an array or a CUDA tensor" % (i, type(im).__name__))
        if not ok or len(shape) != 3 or shape[2] != 3 or shape[0] < 1 or shape[1] < 1:
            raise ValueError("png.encode: image %d is %s %s; only non-empty uint8 (H, W, 3) images are encoded"
                             % (i, dtype, shape))
    if not images:
        return []
    dev = dev or torch.device("cuda", torch.cuda.current_device())
    host_at = {}
    nbytes = 0
    for i, im in enumerate(images):
        if isinstance(im, np.ndarray):
            host_at[i] = nbytes
            nbytes += im.size
    keep, sources, pitches = [], [], []
    if host_at:
        host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        for i, o in host_at.items():
            hv[o:o + images[i].size] = images[i].reshape(-1)
        up = host.to(dev, non_blocking=True)
        keep.append(up)
    for i, im in enumerate(images):
        if i in host_at:
            sources.append(up.data_ptr() + host_at[i])
            pitches.append(3 * im.shape[1])
            continue
        if not (im.stride(2) == 1 and im.stride(1) == 3 and im.stride(0) >= 3 * im.shape[1]):
            im = im.contiguous()
            keep.append(im)
        sources.append(im.data_ptr())
        pitches.append(im.stride(0))
    return encode_at(sources, [tuple(im.shape[:2]) for im in images], pitches, dev)


def encode_at(sources, shapes, pitches, device):
    """The PNG files of images already on ``device`` at addresses ``sources`` with ``(h, w)`` ``shapes`` and row
    ``pitches``: one launch, one read of the sizes, one copy of the files."""
    import torch
    table, counts, ws, out_bytes = encode_layout(sources, shapes, pitches)
    out = torch.empty(out_bytes, dtype=torch.uint8, device=device)
    sizes = torch.empty(len(shapes), dtype=torch.int64, device=device)
    encode_launch(table, counts, ws, out, sizes)
    return download_files(out, sizes)
