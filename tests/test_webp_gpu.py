"""GPU tests of the device WebP decoder: cpb200_webp_decode_batch against cv2.imdecode over lossy files of many sizes
and qualities in one launch, its status on partitions that run out of data, and MultiPoseDetector.run_images on WebP
paths against run_images on the cv2.imread arrays."""
import struct

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import webp
from tests.test_jpeg_cpu import encode, make_image
from tests.test_jpeg_gpu import _detector
from tests.test_png_cpu import write_png, samples
from tests.test_webp_cpu import chunk, cv2_decode, lossy, riff, vp8_chunk, vp8x, with_exif
from tests.webp_writer import matrix as writer_matrix

pytestmark = pytest.mark.gpu
CPB200_ERR_ARG = 1
SIZES = [(1, 1), (17, 1), (17, 15), (16, 16), (33, 17), (3, 130), (37, 53), (64, 96)]


def _launch(src, table, B, ws, ws_bytes, dst, status):
    from centerpose_b200 import _lib
    return _lib.lib().cpb200_webp_decode_batch(src, table, B, ws, ws_bytes, dst, status,
                                               torch.cuda.current_stream().cuda_stream)


def _decode(datas):
    """One launch over all files; returns (images, status) after checking the bytes behind the last image were left
    alone."""
    from centerpose_b200 import _lib
    infos = [webp.parse(d) for d in datas]
    assert all(i.eligible for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = webp.pack(infos, datas, offs[:-1])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((int(offs[-1]) + 256,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(datas),), -1, dtype=torch.int32, device="cuda")
    _lib.launch("webp_decode_batch", src.device, src, src, len(datas), ws, ws_bytes, dst, status)
    out = dst.cpu().numpy()
    assert (out[offs[-1]:] == 77).all()
    return [out[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3) for n, i in enumerate(infos)], status.cpu().numpy()


def matrix():
    """Lossy files from cv2 at qualities 1, 50, 75 and 100 over small and odd sizes and three contents, COCO-sized ones
    at 75 and 95, all eight EXIF orientations, and the extended container with other chunks around the image."""
    files = []
    for k, (h, w) in enumerate(SIZES):
        for q in (1, 50, 75, 100):
            for content in ("noise", "smooth", "smooth_noise"):
                files.append(lossy(h, w, 10 * k + q, q, content))
    for k, (h, w) in enumerate([(480, 640), (640, 480), (427, 640)]):
        for q in (75, 95):
            files.append(lossy(h, w, 100 + k, q))
    for o in range(1, 9):
        files.append(with_exif(lossy(11, 29, o), o, 11, 29))
    files.append(vp8x([chunk(b"ICCP", b"\1\2\3"), vp8_chunk(lossy(40, 70, 3)), chunk(b"XMP ", b"<x/>")], 70, 40, 0x24))
    return files


def test_webp_kernel_equals_cv2_imread():
    files = matrix()
    got, status = _decode(files)
    assert (status == 0).all(), np.flatnonzero(status)
    bad = [n for n, (g, d) in enumerate(zip(got, files)) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, (len(bad), bad[:10])


def test_webp_kernel_equals_cv2_on_writer_files():
    """The writer matrix (both filter types, every sharpness, loop-filter deltas, 1-4 segments absolute and relative,
    1/2/4/8 token partitions, probability updates, skip on and off, every 4x4 mode context, quantiser extremes with
    every delta, 1x1 to 130x3), with cv2-written files around it, in one launch."""
    named = [(name, f.encode()) for name, f in writer_matrix()]
    files = [lossy(33, 17, 1)] + [d for _, d in named] + [lossy(480, 640, 2)]
    got, status = _decode(files)
    assert (status == 0).all(), np.flatnonzero(status)
    bad = [name for (name, d), g in zip(named, got[1:-1]) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, bad
    assert np.array_equal(got[0], cv2_decode(files[0])) and np.array_equal(got[-1], cv2_decode(files[-1]))


def test_webp_batched_equals_single_image_calls():
    files = matrix()[::13]
    batched, _ = _decode(files)
    for d, b in zip(files, batched):
        single, status = _decode([d])
        assert status[0] == 0 and np.array_equal(single[0], b)


def _truncated():
    """Files whose token partition is cut short by k bytes (chunk and RIFF sizes kept consistent), in the simple
    container and in the extended one with an XMP chunk after the image, which libwebp reads as more partition data."""
    out = []
    for h, w, q in ((37, 53, 75), (64, 96, 95)):
        payload = vp8_chunk(lossy(h, w, 7, q))[8:]
        payload = payload[:struct.unpack_from("<I", lossy(h, w, 7, q), 16)[0]]
        for cut in (1, 2, 3, 5, 9, 17, 40, 120):
            p = payload[:-cut]
            out.append(riff(chunk(b"VP8 ", p)))
            out.append(vp8x([chunk(b"VP8 ", p), chunk(b"XMP ", bytes(range(256)) * 2)], w, h))
    return out


def test_truncated_partitions_set_status_where_cv2_fails():
    good = [lossy(20, 30, 1), lossy(33, 17, 2, 95)]
    cut = _truncated()
    fails = [cv2_decode(d) is None for d in cut]
    assert any(fails) and not all(fails)
    files = good[:1] + cut + good[1:]
    got, status = _decode(files)
    assert status[0] == 0 and status[-1] == 0
    for n, (d, g) in enumerate(zip(files, got)):
        want = cv2_decode(d)
        if want is None:
            assert status[n] == 1 and (g == 77).all(), n     # a refused image's slot is left unwritten
        else:
            assert status[n] == 0 and np.array_equal(g, want), n


def test_webp_rejects_host_checkable_arguments():
    from centerpose_b200 import _lib
    data = lossy(16, 16, 1)
    info = webp.parse(data)
    buf, ws_bytes = webp.pack([info], [data], [0])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((16 * 16 * 3,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    s, w, d, st = src.data_ptr(), ws.data_ptr(), dst.data_ptr(), status.data_ptr()
    for args in ((s, s, 0, w, ws_bytes, d, st), (s, s, 65536, w, ws_bytes, d, st), (None, s, 1, w, ws_bytes, d, st),
                 (s, None, 1, w, ws_bytes, d, st), (s, s, 1, None, ws_bytes, d, st), (s, s, 1, w, ws_bytes, None, st),
                 (s, s, 1, w, ws_bytes, d, None)):
        assert _launch(*args) == CPB200_ERR_ARG, args
        assert b"webp_decode_batch" in _lib.lib().cpb200_last_error()
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 77).all() and status.item() == -1
    assert _launch(s, s, 1, w, ws_bytes - 1, d, st) == 0
    assert status.item() == 2 and (dst.cpu().numpy() == 77).all()
    assert _launch(s, s, 1, w, ws_bytes, d, st) == 0
    assert status.item() == 0 and np.array_equal(dst.cpu().numpy().reshape(16, 16, 3), cv2_decode(data))


def _write(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(bytes(data))
    return p


def _webp_paths(tmp_path):
    im = make_image(60, 80, "smooth_noise", 9)
    files = [lossy(120, 160, 1), lossy(100, 150, 2, 95, "smooth"), with_exif(lossy(70, 110, 3, 50), 6, 70, 110),
             cv2.imencode(".webp", im)[1].tobytes(),                                           # lossless: host
             cv2.imencode(".webp", np.dstack([im, im[:, :, 0]]), [cv2.IMWRITE_WEBP_QUALITY, 80])[1].tobytes()]  # alpha
    return [_write(tmp_path, "w%d.webp" % n, d) for n, d in enumerate(files)]


@pytest.fixture
def webp_on_device(monkeypatch):
    """run_images sends WebP files to the device from the first one, so that calls with a few files test that path."""
    from centerpose_b200 import detector
    monkeypatch.setattr(detector, "WEBP_DEVICE_MIN_IMAGES", 1)


def _count_launches(monkeypatch, mod):
    packed = []
    pack = mod.pack
    monkeypatch.setattr(mod, "pack", lambda infos, *a, **k: packed.append(len(infos)) or pack(infos, *a, **k))
    return packed


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_run_images_webp_paths_equal_run_images_arrays(tmp_path, precision, webp_on_device, monkeypatch):
    """The same float rows from WebP paths (lossy ones decoded on the device, a lossless and an alpha file through
    cv2.imread, a truncated file the device refuses and cv2.imread reads), mixed with a JPEG path and an array, as from
    the cv2.imread arrays."""
    packed = _count_launches(monkeypatch, webp)
    det = _detector("dla_34", precision, None)
    paths = _webp_paths(tmp_path)
    readable = [d for d in _truncated() if cv2_decode(d) is not None and webp.parse(d).eligible]
    paths.append(_write(tmp_path, "cut.webp", readable[0]))
    jp = _write(tmp_path, "j.jpg", encode(make_image(120, 160, "noise", 9), 90, "420"))
    inputs = paths + [jp, make_image(80, 100, "smooth", 11)]
    got = det.run_images(inputs)
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    det.device_preprocess = False
    host = det.run_images(inputs)
    det.device_preprocess = True
    for n in range(len(inputs)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n
        assert np.array_equal(host[n], want[n]), n
    assert packed == [4]                             # the three lossy files and the cut one went to the device


def test_run_images_mixed_jpeg_png_webp(tmp_path, webp_on_device, monkeypatch):
    from centerpose_b200 import detector, png
    monkeypatch.setattr(detector, "PNG_DEVICE_MIN_IMAGES", 1)
    packed_png, packed_webp = _count_launches(monkeypatch, png), _count_launches(monkeypatch, webp)
    det = _detector("dla_34", "fp16x2", None)
    w = _webp_paths(tmp_path)[:2]
    inputs = [w[0], _write(tmp_path, "a.jpg", encode(make_image(90, 120, "noise", 1), 85, "420")),
              _write(tmp_path, "b.png", write_png(samples(70, 90, 2, 8, 2), 2, 8)), w[1],
              make_image(64, 80, "smooth", 3)]
    got = det.run_images(inputs)
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    for n in range(len(inputs)):
        assert np.array_equal(got[n], want[n]), n
    assert packed_png == [1] and packed_webp == [2]


def test_run_images_keeps_a_few_webp_files_on_the_host(tmp_path, monkeypatch):
    from centerpose_b200 import detector
    packed = _count_launches(monkeypatch, webp)
    det = _detector("dla_34", "fp16x2", None)
    paths = _webp_paths(tmp_path)[:2]
    want = det.run_images([cv2.imread(p) for p in paths])
    got = det.run_images(paths)
    assert packed == [] and detector.WEBP_DEVICE_MIN_IMAGES > len(paths)
    monkeypatch.setattr(detector, "WEBP_DEVICE_MIN_IMAGES", len(paths))
    got_device = det.run_images(paths)
    assert packed == [len(paths)]
    for n in range(len(paths)):
        assert np.array_equal(got[n], want[n]) and np.array_equal(got_device[n], want[n]), n
