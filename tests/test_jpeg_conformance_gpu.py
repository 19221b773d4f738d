"""GPU conformance tests of the device JPEG decoder on files from tests/jpeg_writer.py: every file of the writer's
corpus the parser sends to the device, sequential and progressive in one launch, against cv2.imdecode on this machine
(never stored bytes: cv2's output outside the IDCT range depends on the host's SIMD path); single-file launches;
``load_images_device`` against cv2.imread on the files on disk; and run_images on COCO-sized writer files."""
import cv2
import numpy as np
import pytest

from centerpose_b200 import jpeg
from tests import jpeg_writer as jw
from tests.test_jpeg_cpu import cv2_decode
from tests.test_jpeg_gpu import _detector
from tests.test_jpeg_progressive_gpu import _decode

pytestmark = pytest.mark.gpu
STATUS = {"device": 0, "range": 1, "corrupt": 1, "no_eoi": 1}


def _device_cases():
    return [c for c in jw.corpus() if c.route in STATUS]


def test_corpus_in_one_launch_equals_cv2_imdecode():
    """One launch over every device-route file: status 0 exactly on the files the corpus expects the device to
    decode, and those equal cv2.imdecode byte for byte; status 1 on out-of-range blocks and corrupt entropy data."""
    cases = _device_cases()
    assert len(cases) >= 100
    got, status = _decode([c.data for c in cases])
    wrong = [(c.name, int(s)) for c, s in zip(cases, status) if s != STATUS[c.route]]
    assert not wrong, wrong
    differ = [c.name for c, g, s in zip(cases, got, status) if s == 0 and not np.array_equal(g, cv2_decode(c.data))]
    assert not differ, differ


@pytest.mark.parametrize("progressive", [False, True])
def test_bad_entropy_data_and_missing_eoi_set_status_and_spare_neighbours(progressive):
    """cv2.imencode files with an undefined Huffman code in the first scan, cut inside the last scan with EOI after the
    cut, and cut before EOI, among good files in one launch: status 1 for those three only, and the good files equal
    cv2.imdecode byte for byte."""
    from tests.test_jpeg_cpu import CONTENTS, encode, make_image
    good = [encode(make_image(64, 80, c, 3), 90, s, progressive=progressive) for c in CONTENTS for s in ("420", "444")]
    data = encode(make_image(96, 128, "noise", 9), 95, "420", progressive=progressive)
    sos = data.rindex(b"\xFF\xDA")
    bad = [jw.corrupt_entropy(data), data[:(sos + len(data)) // 2] + b"\xFF\xD9", data[:-2]]
    files = good[:2] + bad[:1] + good[2:4] + bad[1:] + good[4:]
    got, status = _decode(files)
    assert status.tolist() == [0, 0, 1, 0, 0, 1, 1, 0, 0]
    for n, (d, g) in enumerate(zip(files, got)):
        if status[n] == 0:
            assert np.array_equal(g, cv2_decode(d)), n


def test_single_file_launches_equal_the_batched_launch():
    cases = _device_cases()
    batched, status = _decode([c.data for c in cases])
    for n in list(range(0, len(cases), 7)) + [n for n, c in enumerate(cases) if c.route != "device"][::3]:
        single, st = _decode([cases[n].data])
        assert st[0] == status[n], cases[n].name
        if st[0] == 0:
            assert np.array_equal(single[0], batched[n]), cases[n].name


def test_load_images_device_equals_cv2_imread(tmp_path):
    """Every corpus file from disk: the image cv2.imread gives, whatever the route (device, flagged and read on the
    host, host, refused by the parser), or FileNotFoundError where cv2.imread returns None."""
    from centerpose_b200.detector import load_images_device
    paths, want, unreadable = [], [], []
    for c in jw.corpus():
        p = str(tmp_path / (c.name + ".jpg"))
        with open(p, "wb") as f:
            f.write(c.data)
        im = cv2.imread(p)
        (unreadable if im is None else paths).append(p)
        if im is not None:
            want.append(im)
    assert len(unreadable) >= 12 and len(paths) >= 100
    views, _, _ = load_images_device(paths)
    for p, v, w in zip(paths, views, want):
        assert tuple(v.shape) == w.shape and np.array_equal(v.cpu().numpy(), w), p
    for p in unreadable:
        with pytest.raises(FileNotFoundError):
            load_images_device([paths[0], p])


def _coco_files(tmp_path):
    """COCO-sized writer files: long-code tables with a restart interval that does not divide the MCU row, 16-bit
    DQT with tables after SOF and fill bytes, a custom progressive script with per-scan tables, grayscale declared
    (2, 2)."""
    rng = np.random.RandomState(7)
    frames = [
        jw._frame(rng, jw._ycc((2, 2)), 480, 640, 90, huff="long", ri=7, sof=0xC1),
        jw._frame(rng, jw._ycc((2, 1), ids=(9, 8, 200)), 427, 640, 95, huff="optimal", qt16=True,
                  tables_after_sof=True, fill=True, extras=True),
        jw._frame(rng, jw._ycc((1, 2)), 640, 480, 85, huff="optimal", sof=0xC2, dht_per_scan=True, ri=13,
                  script=[([0, 1, 2], 0, 0, 0, 2), ([0], 1, 9, 0, 1), ([1], 1, 63, 0, 0), ([2], 1, 63, 0, 0),
                          ([0], 10, 63, 0, 1), ([0, 1, 2], 0, 0, 2, 1), ([0, 1, 2], 0, 0, 1, 0), ([0], 1, 63, 1, 0)]),
        jw._frame(rng, [(5, 2, 2, 2, 3, 1)], 480, 640, 80, huff="long", sof=0xC1, ri=40),
    ]
    paths = []
    for n, f in enumerate(frames):
        data = f.encode()
        info = jpeg.parse(data)
        assert info.eligible or info.progressive, info.reason
        paths.append(str(tmp_path / ("coco%d.jpg" % n)))
        with open(paths[-1], "wb") as fh:
            fh.write(data)
    return paths


def test_run_images_writer_paths_equal_run_images_arrays(tmp_path, monkeypatch):
    """run_images on COCO-sized writer files by path (decoded on the device) gives the rows of run_images on the
    cv2.imread arrays, and no file falls back to cv2.imread."""
    from centerpose_b200.detector import load_images_device
    det = _detector("dla_34", "fp16x2", None)
    paths = _coco_files(tmp_path)
    arrays = [cv2.imread(p) for p in paths]
    views, _, _ = load_images_device(paths)
    for v, a in zip(views, arrays):
        assert np.array_equal(v.cpu().numpy(), a)
    want = det.run_images(arrays)
    read = []
    imread = cv2.imread
    monkeypatch.setattr(cv2, "imread", lambda p, *a: read.append(p) or imread(p, *a))
    got = det.run_images(paths)
    assert read == []
    for n in range(len(paths)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n
