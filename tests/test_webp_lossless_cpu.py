"""CPU tests of the lossless WebP host side: which files webp_lossless.parse sends to the device and why the others
stay with cv2.imread or raise (each held against cv2 itself), the launch layout of webp_lossless.pack, the C struct,
the VP8L constant tables of csrc/webp_lossless.cu against their Python copy, and the test-side writer and model that
the GPU tests rely on."""
import os
import re
import struct

import cv2
import numpy as np
import pytest

from centerpose_b200 import webp, webp_lossless
from tests import vp8l_model, vp8l_writer
from tests.test_jpeg_cpu import make_image
from tests.test_webp_cpu import chunk, cv2_decode, riff, tiff, vp8x

ROOT = os.path.dirname(os.path.abspath(__file__)) + "/.."


def lossless(h, w, seed, content="smooth_noise", alpha=False):
    """A simple-container lossless file written by cv2.imencode with no parameters."""
    im = make_image(h, w, content, seed)
    if alpha:
        im = np.dstack([im, make_image(h, w, "noise", seed + 1)[:, :, 0]])
    data = cv2.imencode(".webp", im)[1].tobytes()
    assert data[12:16] == b"VP8L"
    return data


def vp8l_chunk(data):
    ln = struct.unpack_from("<I", data, 16)[0]
    return data[12:20 + ln + (ln & 1)]


def with_exif(data, orientation, h, w):
    return vp8x([vp8l_chunk(data), chunk(b"EXIF", tiff(orientation))], w, h, webp.VP8X_EXIF)


def test_simple_and_extended_files_are_eligible():
    data = lossless(37, 53, 1)
    info = webp_lossless.parse(data)
    assert info.eligible and (info.h, info.w, info.oh, info.ow, info.orientation) == (37, 53, 37, 53, 1)
    assert info.vp8l == 20 and info.stream_bytes() == len(data) - 20
    assert not webp.parse(data).eligible and "lossless" in webp.parse(data).reason
    ext = vp8x([chunk(b"ICCP", b"\1\2\3"), vp8l_chunk(data), chunk(b"XMP ", b"<x/>"), chunk(b"ABCD", b"odd")], 53, 37,
               0x20 | 0x04)
    info = webp_lossless.parse(ext)
    assert info.eligible and (info.oh, info.ow) == (37, 53)
    assert np.array_equal(cv2_decode(ext), cv2_decode(data))


def test_exif_orientation_is_read_as_cv2_reads_it():
    data = lossless(11, 29, 2)
    base = cv2_decode(data)
    for o in range(1, 9):
        f = with_exif(data, o, 11, 29)
        info = webp_lossless.parse(f)
        assert info.eligible and info.orientation == o
        assert cv2_decode(f).shape == (info.oh, info.ow, 3)
    assert np.array_equal(cv2_decode(with_exif(data, 6, 11, 29)), np.rot90(base, -1))
    unflagged = vp8x([vp8l_chunk(data), chunk(b"EXIF", tiff(6))], 29, 11, 0)
    assert webp_lossless.parse(unflagged).orientation == 1 and np.array_equal(cv2_decode(unflagged), base)


def test_host_side_files_have_a_reason():
    data = lossless(20, 30, 3)
    cases = {"animated": vp8x([chunk(b"ANIM", b"\0" * 6), vp8l_chunk(data)], 30, 20, 0x02),
             "RIFF size": data + b"\0\0"}
    for key, f in cases.items():
        info = webp_lossless.parse(f)
        assert not info.eligible and key.lower() in info.reason.lower(), (key, info.reason)
    assert cv2_decode(cases["RIFF size"]) is not None


def test_unreadable_files_raise_where_cv2_refuses():
    data = lossless(20, 30, 4)
    v = vp8l_chunk(data)
    payload = v[8:8 + struct.unpack_from("<I", v, 4)[0]]
    bad = {"signature": riff(chunk(b"VP8L", b"\x2e" + payload[1:])),
           "version": riff(chunk(b"VP8L", payload[:4] + bytes([payload[4] | 0x20]) + payload[5:])),
           "canvas": vp8x([v], 31, 20),
           "past the end": data[:-3],
           "short chunk": riff(chunk(b"VP8L", payload[:4])),
           "no image": riff(chunk(b"XMP ", b"<x/>")),
           "tiny": riff(chunk(b"VP8L", b"\x2f\0\0\0\0\0\0\0"))}
    for name, f in bad.items():
        with pytest.raises(ValueError, match="^" + name):
            webp_lossless.parse(f, name)
        assert cv2_decode(f) is None, name
    with pytest.raises(ValueError, match="no VP8L"):                 # a lossy file is not this parser's
        webp_lossless.parse(cv2.imencode(".webp", make_image(8, 8, "noise", 1), [cv2.IMWRITE_WEBP_QUALITY, 50])[1])


def test_pack_layout():
    datas = [lossless(16, 16, 5), lossless(17, 33, 6), with_exif(lossless(9, 21, 7), 6, 9, 21)]
    infos = [webp_lossless.parse(d) for d in datas]
    buf, ws = webp_lossless.pack(infos, datas, [0, 768, 5000])
    table = buf[:3 * 56].view(webp_lossless.WEBP_LOSSLESS_IMAGE)
    assert ws == sum(i.workspace_bytes() for i in infos)
    assert table["ws_offset"].tolist() == [0, infos[0].workspace_bytes(), infos[0].workspace_bytes() +
                                           infos[1].workspace_bytes()]
    assert table["dst_offset"].tolist() == [0, 768, 5000] and table["orientation"].tolist() == [1, 1, 6]
    assert table["h"].tolist() == [16, 17, 9] and table["w"].tolist() == [16, 33, 21]
    for e, d, i in zip(table, datas, infos):
        o, n = int(e["src_offset"]), int(e["src_bytes"])
        assert o % 16 == 0 and n == len(d) - i.vp8l
        assert bytes(buf[o:o + n]) == d[i.vp8l:] and not buf[o + n:o + n + webp.STREAM_PAD].any()
    # header, two planes, sub-images, 64 groups of 8992 bytes
    assert infos[0].workspace_bytes() == 128 + 2 * 1024 + 4 * (3 * 16 + 256) + 64 * 8992
    with pytest.raises(ValueError):
        webp_lossless.pack([webp_lossless.parse(datas[0] + b"\0\0")], [datas[0] + b"\0\0"], [0])


def test_header_struct_and_budget():
    src = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    body = src[src.index("typedef struct cpb200_webp_lossless_image"):src.index("} cpb200_webp_lossless_image;")]
    fields = [(ln.split()[0], n.strip()) for ln in body.splitlines()[1:] if ln.strip().startswith(("int64_t", "int32_t"))
              for n in ln.split(None, 1)[1].split(";")[0].split(",")]
    assert sum({"int64_t": 8, "int32_t": 4}[t] for t, _ in fields) == webp_lossless.WEBP_LOSSLESS_IMAGE.itemsize == 56
    assert list(webp_lossless.WEBP_LOSSLESS_IMAGE.names) == [n for _, n in fields]
    assert "#define CPB200_WEBP_LOSSLESS_MAX_GROUPS %d" % webp_lossless.MAX_GROUPS in src
    cu = open(os.path.join(ROOT, "centerpose_b200", "csrc", "webp_lossless.cu")).read()
    assert "sizeof(cpb200_webp_lossless_image) == 56" in cu
    assert "kGroupBytes == %d" % webp_lossless.GROUP_BYTES in cu and webp_lossless.GROUP_BYTES == 8992


def _cu_table(src, name):
    m = re.search(r"__constant__ (?:un)?signed char %s\[\d+\] = \{(.*?)\};" % name, src, re.S)
    return [int(v) for v in re.findall(r"-?\d+", m.group(1))]


def test_constant_tables_match_python_copy():
    src = open(os.path.join(ROOT, "centerpose_b200", "csrc", "webp_lossless.cu")).read()
    assert _cu_table(src, "kCodeLengthOrder") == list(vp8l_model.CODE_LENGTH_ORDER)
    assert _cu_table(src, "kDistanceMap") == [v for xy in vp8l_model.DISTANCE_MAP for v in xy]
    # RFC 9649 4.2.2 lists the codes by growing distance from the pixel: the first four are the neighbours
    assert vp8l_model.DISTANCE_MAP[:4] == ((0, 1), (1, 0), (1, 1), (-1, 1)) and len(set(vp8l_model.DISTANCE_MAP)) == 120


@pytest.mark.parametrize("h, w, content, alpha", [(1, 1, "noise", False), (17, 15, "smooth", True),
                                                  (37, 53, "smooth_noise", False), (64, 96, "noise", True),
                                                  (3, 130, "smooth", False)])
def test_model_equals_cv2_on_cv2_files(h, w, content, alpha):
    data = lossless(h, w, h + w, content, alpha)
    info = webp_lossless.parse(data)
    assert np.array_equal(vp8l_model.to_bgr(vp8l_model.decode(data[info.vp8l:])), cv2_decode(data))


def test_model_refuses_truncations_exactly_where_cv2_does():
    """Cut the VP8L payload by k bytes (chunk and RIFF sizes fixed up), in the simple container and in the extended
    one with an XMP chunk after the image, whose bytes libwebp reads as more stream."""
    seen = set()
    for h, w, content in ((37, 53, "smooth_noise"), (20, 30, "noise"), (2, 3, "smooth")):
        data = lossless(h, w, 5, content)
        v = vp8l_chunk(data)
        payload = v[8:8 + struct.unpack_from("<I", v, 4)[0]]
        for cut in range(0, min(len(payload) - 5, 24)):
            p = payload[:len(payload) - cut]
            for f in (riff(chunk(b"VP8L", p)), vp8x([chunk(b"VP8L", p), chunk(b"XMP ", bytes(range(256)))], w, h)):
                want = cv2_decode(f)
                try:
                    info = webp_lossless.parse(f)
                except ValueError:
                    assert want is None
                    continue
                try:
                    got = vp8l_model.to_bgr(vp8l_model.decode(f[info.vp8l:]))
                except vp8l_model.Refused:
                    got = None
                assert (got is None) == (want is None), (h, w, cut)
                assert want is None or np.array_equal(got, want)
                seen.add(want is None)
    assert seen == {True, False}


def test_writer_files_decode_to_the_written_pixels():
    """Every writer file is one the device takes, and cv2.imdecode and the model both give the pixels it wrote."""
    bad = []
    for name, f, expected in vp8l_writer.matrix():
        info = webp_lossless.parse(f, name)
        assert info.eligible and (info.h, info.w) == expected.shape, name
        want = cv2_decode(f)
        model = vp8l_model.decode(f[info.vp8l:])
        if want is None or not np.array_equal(want, vp8l_model.to_bgr(expected)) or not np.array_equal(model, expected):
            bad.append(name)
    assert not bad, bad


def test_writer_matrix_reaches_every_branch():
    names = [n for n, _, _ in vp8l_writer.matrix()]
    files = {n: f for n, f, _ in vp8l_writer.matrix()}
    assert {"cache_%d" % b for b in range(1, 12)} <= set(names)
    assert {"palette_2_0", "palette_3_1", "palette_4_0", "palette_11_5", "palette_16_0", "palette_200_56",
            "palette_256_0"} <= set(names)
    assert vp8l_model.groups(files["groups_64"][20:]) == webp_lossless.MAX_GROUPS
    assert vp8l_model.groups(files["groups_65"][20:]) == webp_lossless.MAX_GROUPS + 1
    assert vp8l_model.groups(files["groups_unused"][20:]) == 4
    # the predictor sub-images of the predictor files, read back from the files, name every mode, 14 and 15 included
    modes = set()
    for name, f in files.items():
        for kind, _, data, _ in vp8l_model.transforms(f[20:]):
            if kind == vp8l_model.PREDICTOR and name.startswith("predictor_"):
                modes |= set(((data >> 8) & 15).tolist())
    assert modes == set(range(16))


def test_writer_codes_use_every_code_length_symbol():
    """The code-length symbols the writer emits over the matrix: every literal length it needs, and 16 (also before
    any non-zero length, where it repeats 8), 17 and 18."""
    seen, first16 = set(), []
    orig = vp8l_writer._tokens

    def spy(lengths, last):
        t = orig(lengths, last)
        seen.update(s for s, _, _ in t)
        nz = [s for s, _, _ in t if s]
        if nz and nz[0] == 16:
            first16.append(True)
        return t
    vp8l_writer._tokens = spy
    try:
        vp8l_writer.matrix()
    finally:
        vp8l_writer._tokens = orig
    assert {16, 17, 18} <= seen and first16


@pytest.mark.parametrize("name, data, reason", vp8l_writer.refused(), ids=[c[0] for c in vp8l_writer.refused()])
def test_writer_refused_streams_are_refused_by_cv2_at_their_check(name, data, reason):
    """Each stream passes the header checks, cv2.imdecode refuses it, and the model refuses it at the check it was
    written to reach."""
    info = webp_lossless.parse(data, name)
    assert info.eligible
    assert cv2_decode(data) is None
    with pytest.raises(vp8l_model.Refused, match=reason):
        vp8l_model.decode(data[info.vp8l:])


def test_copy_at_both_bounds_is_accepted():
    """A backward reference whose distance is every pixel decoded so far and whose length reaches the last pixel."""
    f, expected = {n: (f, e) for n, f, e in vp8l_writer.matrix()}["copy_bounds"]
    assert np.array_equal(cv2_decode(f), vp8l_model.to_bgr(expected))
    assert np.array_equal(vp8l_model.decode(f[20:]), expected)


@pytest.mark.parametrize("tail", [b"XMP " + struct.pack("<I", 100) + b"abc", chunk(b"VP8X", b"\0" * 10)],
                         ids=["chunk past the end", "second VP8X"])
def test_bad_chunk_after_the_image(tail):
    """libwebp never reads the chunks after the image: cv2.imread reads the file, without its EXIF orientation.
    webp.parse still declines it as lossless, webp_lossless.parse takes it."""
    data = lossless(20, 30, 1)
    body = vp8x([vp8l_chunk(data), chunk(b"EXIF", tiff(6))], 30, 20, webp.VP8X_EXIF)[12:] + tail
    f = b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WEBP" + body
    assert "lossless" in webp.parse(f).reason
    info = webp_lossless.parse(f)
    assert info.eligible and info.orientation == 1 and (info.oh, info.ow) == (20, 30)
    assert np.array_equal(cv2_decode(f), cv2_decode(data))
    lossy_body = vp8x([chunk(b"VP8 ", cv2.imencode(".webp", make_image(20, 30, "noise", 1),
                                                  [cv2.IMWRITE_WEBP_QUALITY, 75])[1].tobytes()[20:])], 30, 20)[12:] + tail
    with pytest.raises(ValueError):                   # the lossy parser keeps raising here, as it did
        webp.parse(b"RIFF" + struct.pack("<I", 4 + len(lossy_body)) + b"WEBP" + lossy_body)
