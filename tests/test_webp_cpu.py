"""CPU tests of the WebP host side: which files webp.parse sends to the device and why the others stay with
cv2.imread (checked against cv2 itself), the launch layout of webp.pack, the C struct, and the VP8 constant tables of
csrc/webp.cu against their Python copy."""
import os
import re
import struct

import cv2
import numpy as np
import pytest

from centerpose_b200 import webp
from tests import vp8_tables, webp_model, webp_writer
from tests.test_jpeg_cpu import make_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cv2_decode(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def lossy(h, w, seed, quality=75, content="smooth_noise"):
    """A simple-container lossy file (RIFF, WEBP, VP8 ) written by cv2."""
    data = cv2.imencode(".webp", make_image(h, w, content, seed), [cv2.IMWRITE_WEBP_QUALITY, quality])[1].tobytes()
    assert data[12:16] == b"VP8 "
    return data


def chunk(ctype, payload):
    return ctype + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) % 2 else b"")


def riff(body):
    return b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WEBP" + body


def vp8_chunk(data):
    """The VP8 chunk (header and padded payload) of a simple-container file."""
    ln = struct.unpack_from("<I", data, 16)[0]
    return data[12:20 + ln + (ln & 1)]


def vp8x(chunks, w, h, flags=0):
    """An extended-container file: VP8X (canvas w x h, ``flags``) and then ``chunks``."""
    hdr = bytes([flags, 0, 0, 0]) + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little")
    return riff(chunk(b"VP8X", hdr) + b"".join(chunks))


def tiff(orientation, order="<"):
    """A bare TIFF header with one IFD0 entry: the orientation tag."""
    mark = b"II" if order == "<" else b"MM"
    return mark + struct.pack(order + "HIH", 42, 8, 1) + struct.pack(order + "HHIHH", 0x112, 3, 1, orientation, 0) + \
        b"\0" * 4


def with_exif(data, orientation, h, w, order="<"):
    return vp8x([vp8_chunk(data), chunk(b"EXIF", tiff(orientation, order))], w, h, webp.VP8X_EXIF)


def test_simple_and_extended_lossy_files_are_eligible():
    data = lossy(37, 53, 1)
    info = webp.parse(data)
    assert info.eligible and (info.h, info.w, info.oh, info.ow, info.orientation) == (37, 53, 37, 53, 1)
    assert info.vp8 == 20 and info.stream_bytes() == len(data) - 20
    assert info.workspace_bytes() == 16 + 1184 * 4 * 3
    ext = vp8x([chunk(b"ICCP", b"\1\2\3"), vp8_chunk(data), chunk(b"XMP ", b"<x/>"), chunk(b"ABCD", b"odd")], 53, 37,
               0x20 | 0x04)
    info = webp.parse(ext)
    assert info.eligible and (info.oh, info.ow) == (37, 53)
    assert np.array_equal(cv2_decode(ext), cv2_decode(data))


def test_exif_orientation_is_read_as_cv2_reads_it():
    data = lossy(37, 53, 2)
    base = cv2_decode(data)
    for o in range(1, 9):
        for order in "<>":
            f = with_exif(data, o, 37, 53, order)
            info = webp.parse(f)
            assert info.eligible and info.orientation == o
            assert cv2_decode(f).shape == (info.oh, info.ow, 3)
    # EXIF before the image, the first of two EXIF chunks, odd-length chunks padded to even
    v = vp8_chunk(data)
    cases = {6: vp8x([chunk(b"EXIF", tiff(6)), v], 53, 37, webp.VP8X_EXIF),
             3: vp8x([v, chunk(b"EXIF", tiff(3) + b"\0"), chunk(b"EXIF", tiff(6))], 53, 37, webp.VP8X_EXIF),
             # cv2.imread ignores an EXIF chunk without the VP8X flag, and one with an "Exif\0\0" prefix
             1: vp8x([v, chunk(b"EXIF", tiff(6))], 53, 37, 0)}
    cases[-1] = vp8x([v, chunk(b"EXIF", b"Exif\0\0" + tiff(6))], 53, 37, webp.VP8X_EXIF)
    for o, f in cases.items():
        info = webp.parse(f)
        assert info.orientation == max(o, 1), o
        want = {1: base, 3: base[::-1, ::-1], 6: np.rot90(base, -1), -1: base}[o]
        assert np.array_equal(cv2_decode(f), want), o


def test_host_side_files_have_a_reason():
    data = lossy(20, 30, 3)
    v = vp8_chunk(data)
    im = make_image(20, 30, "smooth_noise", 3)
    lossless = cv2.imencode(".webp", im)[1].tobytes()
    alpha = cv2.imencode(".webp", np.dstack([im, im[:, :, 0]]), [cv2.IMWRITE_WEBP_QUALITY, 80])[1].tobytes()
    cases = {"lossless": lossless,
             "alpha": alpha,
             "animated": vp8x([chunk(b"ANIM", b"\0" * 6), v], 30, 20, 0x02),
             "RIFF size": data + b"\0\0"}
    for key, f in cases.items():
        info = webp.parse(f)
        assert not info.eligible and key.lower() in info.reason.lower(), (key, info.reason)
        if key != "animated":
            assert cv2_decode(f) is not None, key           # cv2.imread reads them on the host path
    assert b"ALPH" in alpha and b"VP8L" in lossless


def test_unreadable_files_raise():
    data = lossy(20, 30, 4)
    v = vp8_chunk(data)
    tag = bytearray(data)
    bad = {"signature": b"RIFX" + data[4:],
           "canvas": vp8x([v], 31, 20),
           "truncated": data[:-3],
           "no image": riff(chunk(b"XMP ", b"<x/>")),
           "first chunk": riff(chunk(b"XMP ", b"<x/>") + v)}
    for name, (pos, val) in {"inter frame": (20, tag[20] | 1), "start code": (23, 0x9c), "no show": (20, tag[20] & ~16)}.items():
        t = bytearray(data)
        t[pos] = val
        bad[name] = bytes(t)
    p0 = bytearray(data)                                     # a first partition longer than the chunk
    p0[20:23] = ((len(data) << 5) | (data[20] & 31)).to_bytes(3, "little")
    bad["partition 0"] = bytes(p0)
    for name, f in bad.items():
        with pytest.raises(ValueError):
            webp.parse(f, name)
        assert cv2_decode(f) is None, name                   # cv2.imread refuses them too


def test_pack_layout():
    datas = [lossy(16, 16, 5), lossy(17, 33, 6, 95), with_exif(lossy(9, 21, 7), 6, 9, 21)]
    infos = [webp.parse(d) for d in datas]
    buf, ws = webp.pack(infos, datas, [0, 768, 5000])
    table = buf[:3 * 56].view(webp.WEBP_IMAGE)
    assert ws == sum(i.workspace_bytes() for i in infos)
    assert table["ws_offset"].tolist() == [0, infos[0].workspace_bytes(), infos[0].workspace_bytes() +
                                           infos[1].workspace_bytes()]
    assert table["dst_offset"].tolist() == [0, 768, 5000] and table["orientation"].tolist() == [1, 1, 6]
    assert table["h"].tolist() == [16, 17, 9] and table["w"].tolist() == [16, 33, 21]
    for e, d, i in zip(table, datas, infos):
        o, n = int(e["src_offset"]), int(e["src_bytes"])
        assert o % 16 == 0 and n == len(d) - i.vp8
        assert bytes(buf[o:o + n]) == d[i.vp8:] and not buf[o + n:o + n + webp.STREAM_PAD].any()
    assert int(table[-1]["src_offset"]) + int(table[-1]["src_bytes"]) + webp.STREAM_PAD <= len(buf)
    with pytest.raises(ValueError):
        webp.pack([webp.parse(cv2.imencode(".webp", make_image(8, 8, "noise", 1))[1].tobytes())], [b""], [0])


def test_header_struct_size():
    src = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    body = src[src.index("typedef struct cpb200_webp_image"):src.index("} cpb200_webp_image;")]
    fields = [(ln.split()[0], n.strip()) for ln in body.splitlines()[1:] if ln.strip().startswith(("int64_t", "int32_t"))
              for n in ln.split(None, 1)[1].split(";")[0].split(",")]
    assert sum({"int64_t": 8, "int32_t": 4}[t] for t, _ in fields) == webp.WEBP_IMAGE.itemsize == 56
    assert list(webp.WEBP_IMAGE.names) == [n for _, n in fields]
    cu = open(os.path.join(ROOT, "centerpose_b200", "csrc", "webp.cu")).read()
    assert "sizeof(cpb200_webp_image) == 56" in cu
    assert webp.MB_WORKSPACE == 1184


def _cu_table(src, name):
    m = re.search(r"__constant__ unsigned (?:char|short) %s(?:\[\d+\])+ = \{(.*?)\};" % name, src, re.S)
    return [int(v) for v in re.findall(r"\d+", m.group(1))]


def test_constant_tables_match_python_copy():
    src = open(os.path.join(ROOT, "centerpose_b200", "csrc", "webp.cu")).read()
    for name, py in (("kDcTable", vp8_tables.DC_TABLE), ("kAcTable", vp8_tables.AC_TABLE),
                     ("kCoeffsUpdateProba", vp8_tables.COEFFS_UPDATE_PROBA), ("kCoeffsProba0", vp8_tables.COEFFS_PROBA0),
                     ("kBModesProba", vp8_tables.BMODES_PROBA)):
        assert _cu_table(src, name) == list(py), name
    dc, ac = vp8_tables.DC_TABLE, vp8_tables.AC_TABLE
    assert dc[:8] == (4, 5, 6, 7, 8, 9, 10, 10) and dc[117] == 132 and dc[127] == 157 and ac[127] == 284
    assert all(a < b for a, b in zip(ac, ac[1:])) and all(a <= b for a, b in zip(dc, dc[1:]))
    # the device's y2 AC step (x * 101581) >> 16 is x * 155 / 100 for every table entry
    assert all((x * 101581) >> 16 == x * 155 // 100 for x in ac)
    p0 = np.array(vp8_tables.COEFFS_PROBA0).reshape(4, 8, 3, 11)
    assert p0[0, 1, 0, :7].tolist() == [253, 136, 254, 255, 228, 219, 128] and (p0[0, 0] == 128).all()
    assert (np.array(vp8_tables.COEFFS_UPDATE_PROBA).reshape(4, 8, 3, 11)[0, 0] == 255).all()
    assert list(vp8_tables.BMODES_PROBA[:9]) == [231, 120, 48, 89, 115, 113, 120, 152, 112]


def _writer_files():
    return [(name, f, f.encode()) for name, f in webp_writer.matrix()]


def test_writer_files_model_equals_cv2():
    """Every file of the writer matrix is one the device takes, and the numpy model of the device stages gives
    cv2.imdecode's pixels for it."""
    bad = []
    for name, f, d in _writer_files():
        info = webp.parse(d, name)
        assert info.eligible and (info.h, info.w) == (f.h, f.w), name
        want = cv2_decode(d)
        if want is None or not np.array_equal(webp_model.decode(f), want):
            bad.append(name)
    assert not bad, bad


def test_writer_matrix_reaches_every_branch():
    """The syntax elements the matrix writes, read back from its frames: each branch the decoder has is present."""
    frames = [f for _, f, _ in _writer_files()]
    filt = {(f.simple, f.level) for f in frames}
    assert {(False, 0), (True, 0), (False, 63), (True, 63)} <= filt
    assert {(s, k) for s in (False, True) for k in range(8)} <= {(f.simple, f.sharpness) for f in frames if f.level}
    assert any(f.update_lf_delta and f.ref_deltas[0] and f.mode_deltas[0] and f.simple for f in frames)
    assert any(f.update_lf_delta and f.ref_deltas[0] and f.mode_deltas[0] and not f.simple for f in frames)
    assert {1, 2, 4, 8} <= {1 << f.log2_parts for f in frames}
    assert any(1 << f.log2_parts > (f.h + 15) >> 4 for f in frames)          # partitions no row reads
    seg = [f for f in frames if f.use_segment]
    assert {1, 2, 3, 4} <= {len({mb.segment for mb in f.mbs}) for f in seg if f.update_map}
    assert {True, False} <= {f.absolute for f in seg if f.update_data}
    assert any(f.update_map and not f.update_data for f in seg) and any(f.update_data and not f.update_map for f in seg)
    assert any(f.update_map and None in f.seg_probs for f in seg) and any(not f.update_map for f in seg)
    assert any(f.proba_updates for f in frames)
    assert any(f.skip_prob is not None and any(mb.skip for mb in f.mbs) for f in frames)
    assert any(f.skip_prob is None for f in frames)
    for q0 in (0, 127):
        for k in ("y1dc", "y2dc", "y2ac", "uvdc", "uvac"):
            assert {-15, 15} <= {f.dq.get(k) for f in frames if f.q0 == q0}, (q0, k)
    contexts, edge_modes = set(), set()
    for f in frames:
        mbw, mbh = (f.w + 15) >> 4, (f.h + 15) >> 4
        top = [0] * (4 * mbw)
        for y in range(mbh):
            left = [0] * 4
            for x in range(mbw):
                mb = f.mbs[y * mbw + x]
                edge = "corner" if x == y == 0 else "top" if y == 0 else "left" if x == 0 else "inside"
                edge_modes.add(("uv", mb.uvmode, edge))
                if mb.i4x4:
                    for sy in range(4):
                        for sx in range(4):
                            m = mb.imodes[4 * sy + sx]
                            contexts.add((top[4 * x + sx], left[sy], m))
                            top[4 * x + sx] = left[sy] = m
                else:
                    edge_modes.add(("y", mb.ymode, edge))
                    top[4 * x:4 * x + 4] = [mb.ymode] * 4
                    left = [mb.ymode] * 4
    assert len(contexts) == 1000                                   # every 4x4 mode under every above / left mode
    assert {(p, m, e) for p in ("y", "uv") for m in range(4) for e in ("corner", "top", "left", "inside")} <= edge_modes
    sizes = {(f.h, f.w) for f in frames}
    assert {(1, 1), (1, 17), (15, 17), (16, 16), (17, 33), (130, 3)} <= sizes


def test_bool_encoder_round_trip():
    """The writer's boolean encoder against a direct transcription of RFC 6386 7.3's decoder."""
    rng = np.random.default_rng(7)
    bits, probs = rng.integers(0, 2, 5000), rng.integers(1, 256, 5000)
    e = webp_writer.BoolEncoder()
    for b, p in zip(bits, probs):
        e.put(int(b), int(p))
    data = e.flush()
    value, rng_, bit_count, pos = (data[0] << 8) | data[1], 255, 0, 2
    out = []
    for p in probs:
        split = 1 + (((rng_ - 1) * int(p)) >> 8)
        big = split << 8
        if value >= big:
            out.append(1)
            rng_ -= split
            value -= big
        else:
            out.append(0)
            rng_ = split
        while rng_ < 128:
            value <<= 1
            rng_ <<= 1
            bit_count += 1
            if bit_count == 8:
                bit_count = 0
                value |= data[pos] if pos < len(data) else 0
                pos += 1
    assert out == bits.tolist()
