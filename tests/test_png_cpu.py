"""CPU tests of the device PNG decoder's host side (centerpose_b200/png.py) and of a numpy/zlib model of the device
stages (inflate, unfilter, Adam7 scatter, depth / palette expansion, BGR, EXIF orientation) against cv2.imread.

The files are written here, chunk by chunk: every colour type and bit depth, interlaced or not, the five filter types
forced row by row, stored / fixed-Huffman / dynamic-Huffman deflate blocks."""
import struct
import zlib

import cv2
import numpy as np
import pytest

from centerpose_b200 import png
from tests.test_jpeg_cpu import make_image

COMBOS = [(ct, d) for ct, depths in sorted(png.DEPTHS.items()) for d in depths]
# (70, 9): more than two 32-row groups of the unfilter, whose lane 0 reads the row above from memory
SIZES = [(1, 1), (3, 5), (13, 37), (2, 130), (70, 9)]
BLOCKS = ["stored", "fixed", "dynamic"]


def chunk(ctype, body):
    return struct.pack(">I", len(body)) + ctype + body + struct.pack(">I", zlib.crc32(ctype + body))


def exif(orientation, big_endian=False):
    """eXIf payload: a TIFF header and IFD0 {Orientation: orientation}."""
    o = ">" if big_endian else "<"
    return (b"MM" if big_endian else b"II") + struct.pack(o + "HI", 42, 8) + struct.pack(o + "H", 1) + \
        struct.pack(o + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(o + "I", 0)


def samples(h, w, ct, depth, seed, npal=None):
    """Seeded samples (h, w, channels) below 2^depth; palette indices below 2^depth (some past ``npal``)."""
    rng = np.random.RandomState(seed)
    ch = png.CHANNELS[ct]
    if depth == 8 and ct != 3:
        im = make_image(h, w, ["noise", "smooth", "smooth_noise"][seed % 3], seed)
        im = np.concatenate([im, im[:, :, :1] ^ 0x5A], 2)[:, :, :ch] if ch != 3 else im
        if ch == 1:
            im = im[:, :, :1]
        return im.astype(np.uint16)
    return rng.randint(0, 1 << depth, (h, w, ch)).astype(np.uint16)


def _pack_row(px, depth):
    """One reduced-image row of samples (w, ch) as PNG bytes."""
    flat = px.reshape(-1).astype(np.uint32)
    if depth == 16:
        return flat.astype(">u2").tobytes()
    if depth == 8:
        return flat.astype(np.uint8).tobytes()
    per = 8 // depth
    flat = np.concatenate([flat, np.zeros((-len(flat)) % per, np.uint32)]).reshape(-1, per)
    shifts = np.array([8 - depth * (k + 1) for k in range(per)], np.uint32)
    return (flat << shifts).sum(1).astype(np.uint8).tobytes()


def _filter(rows, bpp, types):
    """Filtered scanlines: each row (bytes) with its filter type byte prepended."""
    out, prior = [], None
    left = lambda v: np.concatenate([np.zeros(bpp, np.int64), v])[:len(v)]
    for row, ft in zip(rows, types):
        r = np.frombuffer(row, np.uint8).astype(np.int64)
        b = prior if prior is not None else np.zeros_like(r)
        a, c = left(r), left(b)
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        pred = [0, a, b, (a + b) >> 1, paeth][ft]
        out.append(bytes([ft]) + ((r - pred) & 255).astype(np.uint8).tobytes())
        prior = r
    return b"".join(out)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else b if pb <= pc else c


def _reduced(px, interlace):
    if not interlace:
        return [px]
    return [px[y0::dy, x0::dx] for x0, y0, dx, dy in png.ADAM7 if px[y0::dy, x0::dx].size]


def compress(raw, block):
    if block == "stored":
        return zlib.compress(raw, 0)
    c = zlib.compressobj(9, zlib.DEFLATED, 15, 9, zlib.Z_FIXED if block == "fixed" else zlib.Z_DEFAULT_STRATEGY)
    return c.compress(raw) + c.flush()


def write_png(px, ct, depth, interlace=0, block="dynamic", filters=None, palette=None, before=b"", after=b"",
              idat_split=0):
    """A PNG of samples ``px`` (h, w, ch).  ``filters``: one filter type per row of each reduced image (cycled), default
    all five in turn.  ``before`` / ``after``: chunks around the IDAT chunks; ``idat_split``: bytes per IDAT chunk."""
    h, w = px.shape[:2]
    bpp = max(1, png.CHANNELS[ct] * depth // 8)
    raw, n = b"", 0
    for sub in _reduced(px, interlace):
        rows = [_pack_row(sub[y], depth) for y in range(sub.shape[0])]
        types = [(filters or [0, 1, 2, 3, 4])[(n + k) % len(filters or [0, 1, 2, 3, 4])] for k in range(len(rows))]
        n += len(rows)
        raw += _filter(rows, bpp, types)
    z = compress(raw, block)
    out = png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, 0, 0, interlace))
    if palette is not None:
        out += chunk(b"PLTE", palette)
    out += before
    step = idat_split or len(z)
    out += b"".join(chunk(b"IDAT", z[i:i + step]) for i in range(0, len(z), step))
    return out + after + chunk(b"IEND", b"")


def palette_for(depth, seed):
    """A seeded palette, shorter than 2^depth for depths above 1 (indices past it decode black)."""
    n = 2 if depth == 1 else (1 << depth) - (1 << depth) // 4 - 1
    return np.random.RandomState(seed + 7).randint(0, 256, 3 * n).astype(np.uint8).tobytes()


def matrix():
    """(name, file) of the seeded matrix: colour type x depth x interlace x block type x size, filters forced."""
    out, seed = [], 0
    for ct, depth in COMBOS:
        for interlace in (0, 1):
            for block in BLOCKS:
                for h, w in SIZES:
                    seed += 1
                    px = samples(h, w, ct, depth, seed)
                    pal = palette_for(depth, seed) if ct == 3 else None
                    out.append(("ct%d_d%d_i%d_%s_%dx%d" % (ct, depth, interlace, block, h, w),
                                write_png(px, ct, depth, interlace, block, palette=pal)))
    return out


def cv2_decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def _unfilter(f, rows, rb, bpp):
    """Filtered bytes (rows x (1 + rb)) -> uint8 (rows, rb)."""
    out = np.zeros((rows, rb), np.int64)
    prior = np.zeros(rb, np.int64)
    for y in range(rows):
        ft = f[y * (rb + 1)]
        assert ft <= 4
        x = f[y * (rb + 1) + 1:(y + 1) * (rb + 1)].astype(np.int64)
        r = out[y]
        if ft in (0, 2):
            r[:] = (x + (prior if ft == 2 else 0)) & 255
        else:
            for i in range(rb):
                a = r[i - bpp] if i >= bpp else 0
                c = prior[i - bpp] if i >= bpp else 0
                pred = a if ft == 1 else (a + prior[i]) >> 1 if ft == 3 else _paeth(a, prior[i], c)
                r[i] = (x[i] + pred) & 255
        prior = r
    return out.astype(np.uint8)


def _unpack(rowsb, pw, depth, ch):
    """uint8 (rows, rb) -> samples (rows, pw, ch) at 8 bits: 16-bit keeps the high byte, 1/2/4-bit stay indices."""
    if depth == 16:
        return rowsb[:, 0::2][:, :pw * ch].reshape(-1, pw, ch)
    if depth == 8:
        return rowsb[:, :pw * ch].reshape(-1, pw, ch)
    bits = np.unpackbits(rowsb, axis=1)[:, :pw * depth].reshape(-1, pw, depth)
    return (bits * (1 << np.arange(depth - 1, -1, -1))).sum(2).astype(np.uint8)[:, :, None]


def orient(im, o):
    """cv2's EXIF orientation of an (h, w, 3) image: transpose for 5..8, then flips."""
    return {1: im, 2: im[:, ::-1], 3: im[::-1, ::-1], 4: im[::-1], 5: im.transpose(1, 0, 2),
            6: im.transpose(1, 0, 2)[:, ::-1], 7: im.transpose(1, 0, 2)[::-1, ::-1],
            8: im.transpose(1, 0, 2)[::-1]}[o]


def model_decode(data):
    """The device stages on the host: BGR uint8, orientation applied."""
    info = png.parse(data)
    assert info.eligible, info.reason
    d = bytes(data)
    f = np.frombuffer(zlib.decompress(b"".join(d[a:b] for a, b in info.idat)), np.uint8)
    assert len(f) == info.filtered_bytes()
    ct, depth, ch = info.color_type, info.depth, png.CHANNELS[info.color_type]
    bpp = max(1, ch * depth // 8)
    full = np.zeros((info.h, info.w, ch), np.uint8)
    pos = 0
    passes = png.ADAM7 if info.interlace else [(0, 0, 1, 1)]
    for x0, y0, dx, dy in passes:
        pw, ph = -(-(info.w - x0) // dx), -(-(info.h - y0) // dy)
        if pw <= 0 or ph <= 0:
            continue
        rb = info.row_bytes(pw)
        rows = _unfilter(f[pos:pos + ph * (rb + 1)], ph, rb, bpp)
        pos += ph * (rb + 1)
        full[y0::dy, x0::dx] = _unpack(rows, pw, depth, ch)
    if ct == 3:
        pal = np.zeros((256, 3), np.uint8)
        p = np.frombuffer(info.palette, np.uint8).reshape(-1, 3)
        pal[:len(p)] = p
        bgr = pal[full[:, :, 0]][:, :, ::-1]
    elif ct in (0, 4):
        g = full[:, :, 0].astype(np.int64) * (255 // ((1 << depth) - 1) if depth < 8 else 1)
        bgr = np.repeat(g.astype(np.uint8)[:, :, None], 3, 2)
    else:
        bgr = full[:, :, 2::-1]
    return np.ascontiguousarray(orient(bgr, info.orientation))


def test_model_equals_cv2_imread_over_the_matrix():
    bad = [name for name, data in matrix() if not np.array_equal(model_decode(data), cv2_decode(data))]
    assert not bad, (len(bad), bad[:10])


@pytest.mark.parametrize("ct,depth", [(2, 8), (0, 16), (3, 4), (6, 16)])
def test_idat_split_over_many_chunks(ct, depth):
    px = samples(19, 23, ct, depth, 5)
    pal = palette_for(depth, 5) if ct == 3 else None
    data = write_png(px, ct, depth, 1, palette=pal, idat_split=7)
    info = png.parse(data)
    assert info.eligible and len(info.idat) > 10
    assert np.array_equal(model_decode(data), cv2_decode(data))


@pytest.mark.parametrize("orientation", range(1, 9))
@pytest.mark.parametrize("where", ["before", "after"])
def test_exif_orientation_before_or_after_idat(orientation, where):
    px = samples(5, 9, 2, 8, orientation)
    data = write_png(px, 2, 8, **{where: chunk(b"eXIf", exif(orientation, orientation % 2 == 0))})
    info = png.parse(data)
    assert info.orientation == orientation
    assert (info.oh, info.ow) == ((9, 5) if orientation >= 5 else (5, 9))
    want = cv2_decode(data)
    assert want.shape == (info.oh, info.ow, 3)
    assert np.array_equal(model_decode(data), want)


def test_first_exif_chunk_wins_and_prefixed_exif_is_ignored():
    px = samples(4, 6, 0, 8, 3)
    data = write_png(px, 0, 8, before=chunk(b"eXIf", exif(3)) + chunk(b"eXIf", exif(6)))
    assert png.parse(data).orientation == 3 and np.array_equal(model_decode(data), cv2_decode(data))
    data = write_png(px, 0, 8, before=chunk(b"eXIf", b"Exif\x00\x00" + exif(3)))
    assert png.parse(data).orientation == 1 and np.array_equal(model_decode(data), cv2_decode(data))


@pytest.mark.parametrize("extra", ["tRNS", "gAMA", "sBIT", "iCCP", "bKGD", "tEXt", "PLTE"])
@pytest.mark.parametrize("ct,depth", [(0, 8), (0, 2), (2, 16), (3, 8), (4, 8), (6, 8)])
def test_ancillary_chunks_change_nothing(extra, ct, depth):
    px = samples(6, 11, ct, depth, ct * 17 + depth)
    pal = palette_for(depth, 1) if ct == 3 else None
    ch = png.CHANNELS[ct]
    body = {"tRNS": b"\x00\x80\x00\x10" if ct == 3 else b"\x00\x01" * (1 if ct == 0 else 3) if ct in (0, 2) else None,
            "gAMA": struct.pack(">I", 100000), "sBIT": bytes([max(1, depth // 2)] * (3 if ct == 3 else ch)),
            "iCCP": b"p\x00\x00" + zlib.compress(b"not a profile" * 8), "bKGD": b"\x00" * (1 if ct == 3 else 2 * (1 if ct in (0, 4) else 3)),
            "tEXt": b"Comment\x00hello", "PLTE": palette_for(8, 2)}[extra]
    if body is None or (extra == "PLTE" and ct in (0, 3, 4)):
        pytest.skip("chunk not allowed for this colour type")
    plain = write_png(px, ct, depth, palette=pal)
    data = write_png(px, ct, depth, palette=pal, before=chunk(extra.encode(), body))
    assert png.parse(data).eligible
    assert np.array_equal(cv2_decode(data), cv2_decode(plain))
    assert np.array_equal(model_decode(data), cv2_decode(data))


def test_palette_shorter_than_the_depth_decodes_black():
    px = np.array([[[0], [1], [2], [255]]], np.uint16)
    data = write_png(px, 3, 8, palette=bytes([10, 20, 30, 40, 50, 60]))
    want = np.array([[[30, 20, 10], [60, 50, 40], [0, 0, 0], [0, 0, 0]]], np.uint8)
    assert np.array_equal(cv2_decode(data), want) and np.array_equal(model_decode(data), want)


def test_sixteen_bit_keeps_the_high_byte_and_gray_expands_by_replication():
    px = np.array([[[0x12FF], [0xFF00], [0x0080], [0x8000]]], np.uint16)
    assert cv2_decode(write_png(px, 0, 16))[0, :, 0].tolist() == [0x12, 0xFF, 0, 0x80]
    for depth in (1, 2, 4):
        px = np.arange(1 << depth, dtype=np.uint16).reshape(1, -1, 1)
        assert cv2_decode(write_png(px, 0, depth))[0, :, 0].tolist() == \
            [v * 255 // ((1 << depth) - 1) for v in range(1 << depth)]


def _apng(default_in_animation):
    """A two-frame APNG whose IDAT image differs from its first animation frame when it is not part of the
    animation."""
    w, h = 4, 2
    f0 = b"".join(b"\x00" + bytes([10 * r + c for c in range(3 * w)]) for r in range(h))
    f1 = b"".join(b"\x00" + bytes([200 + r] * 3 * w) for r in range(h))
    fctl = lambda seq: chunk(b"fcTL", struct.pack(">IIIIIHHBB", seq, w, h, 0, 0, 1, 10, 0, 0))
    out = png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + \
        chunk(b"acTL", struct.pack(">II", 2, 0))
    if default_in_animation:
        out += fctl(0) + chunk(b"IDAT", zlib.compress(f0)) + fctl(1) + \
            chunk(b"fdAT", struct.pack(">I", 2) + zlib.compress(f1))
    else:
        out += chunk(b"IDAT", zlib.compress(f0)) + fctl(0) + \
            chunk(b"fdAT", struct.pack(">I", 1) + zlib.compress(f1)) + fctl(2) + \
            chunk(b"fdAT", struct.pack(">I", 3) + zlib.compress(f1))
    return out + chunk(b"IEND", b""), f0, f1


def test_apng_stays_on_the_host():
    """cv2.imread returns the first animation frame, not the IDAT image when that is outside the animation."""
    for default_in_animation in (True, False):
        data, f0, f1 = _apng(default_in_animation)
        info = png.parse(data)
        assert not info.eligible and "APNG" in info.reason
        got = cv2_decode(data)[:, :, 2]
        first = f0 if default_in_animation else f1
        assert got.tolist() == [list(first[r * 13 + 1:(r + 1) * 13:3]) for r in range(2)]


def _with_chunk_edit(data, ctype, fn):
    i = data.index(ctype) - 4
    n = int.from_bytes(data[i:i + 4], "big")
    return data[:i] + fn(data[i:i + 12 + n]) + data[i + 12 + n:]


def test_parser_rejects_unreadable_files_naming_them():
    good = write_png(samples(8, 8, 2, 8, 1), 2, 8)
    flip_crc = lambda c: c[:-1] + bytes([c[-1] ^ 1])
    cases = {
        "signature": b"\x89PNX" + good[4:],
        "crc": _with_chunk_edit(good, b"IDAT", flip_crc),
        "ancillary crc": write_png(samples(8, 8, 2, 8, 1), 2, 8, before=flip_crc(chunk(b"tEXt", b"a\x00b"))),
        "truncated": good[:-12],
        "truncated inside a chunk": good[:40],
        "unknown critical": write_png(samples(8, 8, 2, 8, 1), 2, 8, before=chunk(b"ABCD", b"xx")),
        "oversize": _with_chunk_edit(good, b"IHDR", lambda c: chunk(b"IHDR", struct.pack(">II", 1 << 31, 8) + c[16:21])),
        "zero width": _with_chunk_edit(good, b"IHDR", lambda c: chunk(b"IHDR", struct.pack(">II", 0, 8) + c[16:21])),
        "bad depth": _with_chunk_edit(good, b"IHDR", lambda c: chunk(b"IHDR", c[8:16] + b"\x04\x02\x00\x00\x00")),
        "interlace 2": _with_chunk_edit(good, b"IHDR", lambda c: chunk(b"IHDR", c[8:20] + b"\x02")),
        "no palette": write_png(samples(8, 8, 3, 8, 1), 3, 8),
        "duplicate palette": write_png(samples(8, 8, 3, 2, 1), 3, 2, palette=palette_for(2, 1),
                                       before=chunk(b"PLTE", palette_for(2, 2))),
    }
    z = compress(_filter([b"\x00" * 24] * 8, 3, [0] * 8), "dynamic")
    cases["IDAT chunks apart"] = png.SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", 8, 8, 8, 2, 0, 0, 0)) + \
        chunk(b"IDAT", z[:5]) + chunk(b"tEXt", b"a\x00b") + chunk(b"IDAT", z[5:]) + chunk(b"IEND", b"")
    for what, data in cases.items():
        with pytest.raises(ValueError, match="img_x.png"):
            png.parse(data, "img_x.png")
        # cv2 refuses each of these too, except an ancillary chunk's CRC error, which libpng only warns about
        if what != "ancillary crc":
            assert cv2_decode(data) is None, what


def test_oversize_images_stay_on_the_host():
    good = write_png(samples(8, 8, 2, 8, 1), 2, 8)
    for w, h in ((png.MAX_DIMENSION + 1, 1), (1 << 15, (1 << 15) + 1)):
        data = _with_chunk_edit(good, b"IHDR", lambda c: chunk(b"IHDR", struct.pack(">II", w, h) + c[16:21]))
        info = png.parse(data)
        assert not info.eligible and "size" in info.reason


def test_pack_lays_out_streams_palettes_and_workspace():
    files = [write_png(samples(9, 13, 3, 4, 2), 3, 4, 1, palette=palette_for(4, 2), idat_split=9),
             write_png(samples(5, 7, 6, 16, 3), 6, 16, before=chunk(b"eXIf", exif(6))),
             write_png(samples(1, 1, 0, 1, 4), 0, 1, block="stored")]
    infos = [png.parse(d) for d in files]
    dst = [0, 1000, 5000]
    buf, ws = png.pack(infos, files, dst)
    table = buf[:len(files) * png.PNG_IMAGE.itemsize].view(png.PNG_IMAGE)
    end = 0
    for e, info, data, o in zip(table, infos, files, dst):
        z = b"".join(data[a:b] for a, b in info.idat)
        s = int(e["src_offset"])
        assert s % 16 == 0 and s >= len(buf[:len(files) * 72]) and e["src_bytes"] == len(z)
        assert buf[s:s + len(z)].tobytes() == z and not buf[s + len(z):s + len(z) + png.STREAM_PAD].any()
        if info.color_type == 3:
            p = int(e["palette_offset"])
            assert p >= s + len(z) + png.STREAM_PAD and p % 16 == 0
            assert buf[p:p + len(info.palette)].tobytes() == info.palette and not buf[p + len(info.palette):p + 768].any()
        assert e["ws_offset"] == end and e["ws_offset"] % 16 == 0
        assert e["ws_bytes"] == info.workspace_bytes() >= info.filtered_bytes() + 16
        end += int(e["ws_bytes"])
        assert e["dst_offset"] == o and (e["h"], e["w"]) == (info.h, info.w)
        assert (e["color_type"], e["depth"], e["interlace"], e["orientation"]) == \
            (info.color_type, info.depth, info.interlace, info.orientation)
    assert ws == end and table[1]["orientation"] == 6
    with pytest.raises(ValueError, match="not eligible"):
        png.pack([png.parse(_apng(True)[0])], [_apng(True)[0]], [0])


def test_header_struct_size():
    src = open(__file__.replace("tests/test_png_cpu.py", "include/centerpose_b200.h")).read()
    body = src[src.index("typedef struct cpb200_png_image"):src.index("} cpb200_png_image;")]
    sizes = {"int64_t": 8, "int32_t": 4}
    total = sum(sizes[t] * len(names.split(","))
                for t, names in [(ln.split()[0], ln.split(None, 1)[1].split(";")[0])
                                 for ln in body.splitlines()[1:] if ln.strip().startswith(("int64_t", "int32_t"))])
    assert total == png.PNG_IMAGE.itemsize == 72
    assert list(png.PNG_IMAGE.names) == [n.strip() for ln in body.splitlines()[1:]
                                         if ln.strip().startswith(("int64_t", "int32_t"))
                                         for n in ln.split(None, 1)[1].split(";")[0].split(",")]
