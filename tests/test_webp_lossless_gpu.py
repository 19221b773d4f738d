"""GPU tests of the device lossless WebP decoder: cpb200_webp_lossless_decode_batch against cv2.imdecode over
cv2-written and writer files in one launch, its status on streams libwebp refuses and on a file over the group budget,
and MultiPoseDetector.run_images on lossless paths against run_images on the cv2.imread arrays."""
import re
import struct

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import webp, webp_lossless
from tests import vp8l_writer
from tests.test_jpeg_cpu import encode, make_image
from tests.test_jpeg_gpu import _detector
from tests.test_png_cpu import samples, write_png
from tests.test_webp_cpu import chunk, cv2_decode, lossy, riff, tiff, vp8x
from tests.test_webp_gpu import _count_launches, _write
from tests.test_webp_lossless_cpu import lossless, vp8l_chunk, with_exif

pytestmark = pytest.mark.gpu
CPB200_ERR_ARG = 1
SIZES = [(1, 1), (1, 17), (17, 1), (17, 15), (16, 16), (33, 17), (3, 130), (37, 53), (64, 96)]


def _launch(src, table, B, ws, ws_bytes, dst, status):
    from centerpose_b200 import _lib
    return _lib.lib().cpb200_webp_lossless_decode_batch(src, table, B, ws, ws_bytes, dst, status,
                                                        torch.cuda.current_stream().cuda_stream)


def _decode(datas):
    """One launch over all files; returns (images, status) after checking the bytes behind the last image were left
    alone."""
    from centerpose_b200 import _lib
    infos = [webp_lossless.parse(d) for d in datas]
    assert all(i.eligible for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = webp_lossless.pack(infos, datas, offs[:-1])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((int(offs[-1]) + 256,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(datas),), -1, dtype=torch.int32, device="cuda")
    _lib.launch("webp_lossless_decode_batch", src.device, src, src, len(datas), ws, ws_bytes, dst, status)
    out = dst.cpu().numpy()
    assert (out[offs[-1]:] == 77).all()
    return [out[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3) for n, i in enumerate(infos)], status.cpu().numpy()


def matrix():
    """cv2.imencode default (lossless) files over small and odd sizes, three contents and BGRA sources, a few-colour
    image (cv2 writes a palette), COCO-sized ones, all eight EXIF orientations and the extended container."""
    files = []
    for k, (h, w) in enumerate(SIZES):
        for content in ("noise", "smooth", "smooth_noise"):
            files.append(lossless(h, w, 10 * k, content))
        files.append(lossless(h, w, 10 * k + 1, "smooth_noise", alpha=True))
    few = (make_image(45, 61, "smooth", 3) // 64 * 64).astype(np.uint8)
    files.append(cv2.imencode(".webp", few)[1].tobytes())
    for k, (h, w) in enumerate([(480, 640), (640, 480), (427, 640)]):
        files.append(lossless(h, w, 100 + k, ("smooth_noise", "smooth", "noise")[k]))
    for o in range(1, 9):
        files.append(with_exif(lossless(11, 29, o), o, 11, 29))
    files.append(vp8x([chunk(b"ICCP", b"\1\2\3"), vp8l_chunk(lossless(40, 70, 3)), chunk(b"XMP ", b"<x/>")], 70, 40,
                      0x24))
    # a chunk past the end after the image: cv2.imread reads the image and drops the EXIF orientation
    body = vp8x([vp8l_chunk(lossless(21, 13, 4)), chunk(b"EXIF", tiff(6))], 13, 21, webp.VP8X_EXIF)[12:] + \
        b"XMP " + struct.pack("<I", 100) + b"abc"
    files.append(b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WEBP" + body)
    return files


def test_lossless_kernel_equals_cv2_imread_with_writer_files():
    """One launch over the cv2 files and the writer matrix (without the file over the group budget)."""
    named = [(name, f) for name, f, _ in vp8l_writer.matrix() if name != "groups_65"]
    files = matrix() + [f for _, f in named]
    got, status = _decode(files)
    assert (status == 0).all(), np.flatnonzero(status)
    bad = [n for n, (g, d) in enumerate(zip(got, files)) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, (len(bad), [named[n - len(files) + len(named)][0] if n >= len(files) - len(named) else n
                                for n in bad[:10]])


def test_batched_equals_single_image_calls():
    files = matrix()[::7]
    batched, _ = _decode(files)
    for d, b in zip(files, batched):
        single, status = _decode([d])
        assert status[0] == 0 and np.array_equal(single[0], b)


def _refused():
    """Files libwebp refuses past the header: truncated streams (sizes fixed up, in the simple container and with an
    XMP chunk after the image), and streams with one byte flipped, which break codes, distances and lengths."""
    out = []
    for h, w in ((37, 53), (20, 30)):
        v = vp8l_chunk(lossless(h, w, 7))
        payload = v[8:8 + struct.unpack_from("<I", v, 4)[0]]
        for cut in (1, 2, 3, 5, 9, 17, 40):
            p = payload[:-cut]
            out.append(riff(chunk(b"VP8L", p)))
            out.append(vp8x([chunk(b"VP8L", p), chunk(b"XMP ", bytes(range(256)))], w, h))
        for k in range(5, len(payload), max(1, len(payload) // 40)):
            p = bytearray(payload)
            p[k] ^= 0x5A
            out.append(riff(chunk(b"VP8L", bytes(p))))
    return [d for d in out if _parses(d)]


def _parses(d):
    try:
        return webp_lossless.parse(d).eligible
    except ValueError:
        return False


def test_status_one_exactly_where_cv2_refuses():
    """Truncated and byte-flipped cv2 files, and the writer's refused streams: each one refused at a single check (a
    backward reference before the image start or past its end, a transform read twice, colour cache bits of 0, 12 or
    15, max_symbol past the alphabet)."""
    good = [lossless(20, 30, 1), lossless(33, 17, 2)]
    bad = _refused()
    fails = [cv2_decode(d) is None for d in bad]
    assert sum(fails) >= 10 and not all(fails)
    written = [f for _, f, _ in vp8l_writer.refused()]
    assert all(cv2_decode(f) is None for f in written)
    files = good[:1] + bad + written + good[1:]
    got, status = _decode(files)
    assert status[0] == 0 and status[-1] == 0
    for n, (d, g) in enumerate(zip(files, got)):
        want = cv2_decode(d)
        if want is None:
            assert status[n] == 1 and (g == 77).all(), n     # a refused image's slot is left unwritten
        else:
            assert status[n] == 0 and np.array_equal(g, want), n
    assert (status[1 + len(bad):1 + len(bad) + len(written)] == 1).all()


def test_over_budget_file_gets_status_two():
    over = {name: f for name, f, _ in vp8l_writer.matrix()}["groups_65"]
    assert cv2_decode(over) is not None
    got, status = _decode([lossless(9, 9, 1), over, lossless(9, 9, 2)])
    assert status.tolist() == [0, 2, 0] and (got[1] == 77).all()


def test_rejects_host_checkable_arguments():
    from centerpose_b200 import _lib
    data = lossless(16, 16, 1)
    info = webp_lossless.parse(data)
    buf, ws_bytes = webp_lossless.pack([info], [data], [0])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((16 * 16 * 3,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    s, w, d, st = src.data_ptr(), ws.data_ptr(), dst.data_ptr(), status.data_ptr()
    for args in ((s, s, 0, w, ws_bytes, d, st), (s, s, 65536, w, ws_bytes, d, st), (None, s, 1, w, ws_bytes, d, st),
                 (s, None, 1, w, ws_bytes, d, st), (s, s, 1, None, ws_bytes, d, st), (s, s, 1, w, ws_bytes, None, st),
                 (s, s, 1, w, ws_bytes, d, None)):
        assert _launch(*args) == CPB200_ERR_ARG, args
        assert b"webp_lossless_decode_batch" in _lib.lib().cpb200_last_error()
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 77).all() and status.item() == -1
    assert _launch(s, s, 1, w, ws_bytes - 1, d, st) == 0
    assert status.item() == 2 and (dst.cpu().numpy() == 77).all()
    assert _launch(s, s, 1, w, ws_bytes, d, st) == 0
    assert status.item() == 0 and np.array_equal(dst.cpu().numpy().reshape(16, 16, 3), cv2_decode(data))


@pytest.fixture
def lossless_on_device(monkeypatch):
    """run_images sends WebP files to the device from the first one, so that calls with a few files test that path."""
    from centerpose_b200 import detector
    monkeypatch.setattr(detector, "WEBP_LOSSLESS_DEVICE_MIN_IMAGES", 1)
    monkeypatch.setattr(detector, "WEBP_DEVICE_MIN_IMAGES", 1)


def _lossless_paths(tmp_path):
    over = {name: f for name, f, _ in vp8l_writer.matrix()}["groups_65"]
    files = [lossless(120, 160, 1), lossless(100, 150, 2, "smooth", alpha=True),
             with_exif(lossless(70, 110, 3), 6, 70, 110), over]
    return [_write(tmp_path, "l%d.webp" % n, d) for n, d in enumerate(files)]


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_run_images_lossless_paths_equal_run_images_arrays(tmp_path, precision, lossless_on_device, monkeypatch):
    """The same float rows from lossless paths (three decoded on the device, one over the group budget read by
    cv2.imread) mixed with a lossy WebP, a JPEG and a PNG path and an array, as from the cv2.imread arrays."""
    from centerpose_b200 import detector, png
    monkeypatch.setattr(detector, "PNG_DEVICE_MIN_IMAGES", 1)
    packed, packed_lossy = _count_launches(monkeypatch, webp_lossless), _count_launches(monkeypatch, webp)
    det = _detector("dla_34", precision, None)
    inputs = _lossless_paths(tmp_path) + [
        _write(tmp_path, "lossy.webp", lossy(90, 120, 4)),
        _write(tmp_path, "j.jpg", encode(make_image(120, 160, "noise", 9), 90, "420")),
        _write(tmp_path, "p.png", write_png(samples(70, 90, 2, 8, 2), 2, 8)),
        make_image(80, 100, "smooth", 11)]
    got = det.run_images(inputs)
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    for n in range(len(inputs)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n
    assert packed == [4] and packed_lossy == [1]


def test_run_images_raises_on_a_corrupt_lossless_file(tmp_path, lossless_on_device, monkeypatch):
    """A file the device refuses (status 1) goes to cv2.imread, which refuses it too: the same FileNotFoundError
    naming the path as with the host decode."""
    packed = _count_launches(monkeypatch, webp_lossless)
    det = _detector("dla_34", "fp16x2", None)
    bad = {name: f for name, f, _ in vp8l_writer.refused()}["distance_before_start"]
    paths = _lossless_paths(tmp_path)[:1] + [_write(tmp_path, "bad.webp", bad)]
    with pytest.raises(FileNotFoundError, match=re.escape(paths[1])):
        det.run_images(paths)
    assert packed == [2]                              # both files went to the device
    det.device_preprocess = False
    with pytest.raises(FileNotFoundError, match=re.escape(paths[1])):
        det.run_images(paths)


def test_run_images_keeps_a_few_lossless_files_on_the_host(tmp_path, monkeypatch):
    from centerpose_b200 import detector
    packed = _count_launches(monkeypatch, webp_lossless)
    det = _detector("dla_34", "fp16x2", None)
    paths = _lossless_paths(tmp_path)[:3]
    want = det.run_images([cv2.imread(p) for p in paths])
    got = det.run_images(paths)
    assert packed == [] and detector.WEBP_LOSSLESS_DEVICE_MIN_IMAGES > len(paths)
    monkeypatch.setattr(detector, "WEBP_LOSSLESS_DEVICE_MIN_IMAGES", len(paths))
    got_device = det.run_images(paths)
    assert packed == [len(paths)]
    for n in range(len(paths)):
        assert np.array_equal(got[n], want[n]) and np.array_equal(got_device[n], want[n]), n
