"""GPU tests of progressive JPEG decoding: cpb200_jpeg_decode_batch on progressive files against cv2.imdecode /
cv2.imread, mixed with sequential files in one launch, its status on bad entropy data, and
MultiPoseDetector.run_images on progressive paths against run_images on the cv2.imread arrays."""
import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import jpeg
from tests.test_jpeg_cpu import CONTENTS, QUALITIES, SAMPLINGS, SIZES, cv2_decode, encode, make_image, with_exif
from tests.test_jpeg_gpu import COCO, _detector, _launch
from tests.test_jpeg_progressive_cpu import RESTARTS, _sos, penc

pytestmark = pytest.mark.gpu


def _decode(datas):
    """One launch over all files, sequential or progressive; returns (images, status) after checking the bytes
    behind the last image were left alone."""
    from centerpose_b200 import _lib
    infos = [jpeg.parse(d) for d in datas]
    assert all(i.eligible or i.progressive for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = jpeg.pack(infos, datas, offs[:-1])
    src = torch.from_numpy(buf).cuda()
    ws = torch.full((ws_bytes,), 0x55, dtype=torch.uint8, device="cuda")      # the kernel must zero the blocks itself
    dst = torch.full((int(offs[-1]) + 256,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((len(datas),), -1, dtype=torch.int32, device="cuda")
    _lib.check(_launch(src.data_ptr(), src.data_ptr(), len(datas), ws.data_ptr(), ws_bytes, dst.data_ptr(),
                       status.data_ptr()), "jpeg_decode_batch")
    out = dst.cpu().numpy()
    assert (out[offs[-1]:] == 77).all()
    return [out[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3) for n, i in enumerate(infos)], status.cpu().numpy()


def _grid_files():
    files = []
    for sampling in SAMPLINGS:
        gray = sampling == "gray"
        for quality in QUALITIES:
            for h, w in SIZES:
                for content in CONTENTS:
                    for rst in RESTARTS:
                        files.append(penc(make_image(h, w, content, h * 7 + w + quality, gray=gray), quality,
                                          sampling, rst))
        for quality in (75, 95):
            for h, w in COCO:
                for content in CONTENTS:
                    files.append(penc(make_image(h, w, content, h + w + quality, gray=gray), quality, sampling))
    return files


def test_progressive_kernel_equals_cv2_imdecode():
    """Sizes 1x1 to 97x131, qualities 10-100, 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 / grayscale, restart intervals 0, 1, 3
    and 100, three contents, plus COCO-sized images, all progressive, in one launch, byte for byte."""
    files = _grid_files()
    assert all(jpeg.parse(d).progressive for d in files)
    got, status = _decode(files)
    assert (status == 0).all(), np.flatnonzero(status)[:10]
    bad = [n for n, (g, d) in enumerate(zip(got, files)) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, (len(bad), bad[:10])


def test_mixed_launch_equals_single_image_launches():
    """Sequential and progressive files alternating in one launch give the images of one launch per file."""
    prog = _grid_files()[::23]
    seq = [encode(make_image(h, w, "smooth_noise", h + w, gray=s == "gray"), 85, s, rst=r)
           for (h, w), s, r in zip(SIZES * 4, list(SAMPLINGS) * 6, [0, 3] * 14)]
    files = [f for pair in zip(prog, seq) for f in pair] + prog[len(seq):]
    batched, status = _decode(files)
    assert (status == 0).all()
    for d, b in zip(files, batched):
        single, st = _decode([d])
        assert st[0] == 0 and np.array_equal(single[0], b)
        assert np.array_equal(b, cv2_decode(d))


def _truncated():
    """A progressive file cut inside the entropy data of its last scan: the parser takes it, the data runs out."""
    data = penc(make_image(96, 128, "noise", 9), 95, "420")
    cut = data[:(_sos(data, 9) + len(data)) // 2]
    assert jpeg.parse(cut).progressive
    return cut


def test_bad_entropy_data_sets_status_and_spares_neighbours():
    good = [penc(make_image(64, 80, c, 3), 90, s) for c in CONTENTS for s in ("420", "444")]
    files = good[:3] + [_truncated()] + good[3:]
    got, status = _decode(files)
    assert status[3] != 0 and (np.delete(status, 3) == 0).all()
    for n, (d, g) in enumerate(zip(files, got)):
        if n != 3:
            assert np.array_equal(g, cv2_decode(d)), n


def _files(tmp_path, specs):
    paths = []
    for n, (h, w, sampling, kw) in enumerate(specs):
        kw = dict(kw)
        orientation = kw.pop("orientation", 0)
        data = encode(make_image(h, w, CONTENTS[n % 3], 200 + n), 90, sampling, **kw)
        if orientation:
            data = with_exif(data, orientation)
        p = str(tmp_path / ("p%d.jpg" % n))
        with open(p, "wb") as f:
            f.write(data)
        paths.append(p)
    return paths


PROG = {"progressive": True}
SPECS = [(120, 160, "420", PROG), (100, 150, "444", PROG), (120, 160, "422", dict(PROG, rst=4)),
         (130, 170, "440", PROG), (160, 120, "420", dict(PROG, orientation=6)), (90, 140, "420", dict(PROG, orientation=3)),
         (110, 150, "420", {}), (100, 150, "411", PROG)]


@pytest.mark.parametrize("precision,scales", [(p, s) for p in ("fp32", "fp16x2") for s in (None, (1, 0.75))])
def test_run_images_progressive_paths_equal_run_images_arrays(tmp_path, monkeypatch, precision, scales):
    """The same float rows from progressive paths (decoded on the device, EXIF orientations among them) as from the
    cv2.imread arrays, with a baseline and a progressive 4:1:1 file (host path) mixed in; cv2.imread is called for the
    4:1:1 file only."""
    det = _detector("dla_34", precision, scales)
    paths = _files(tmp_path, SPECS)
    want = det.run_images([cv2.imread(p) for p in paths])
    read = []
    imread = cv2.imread
    monkeypatch.setattr(cv2, "imread", lambda p, *a: read.append(p) or imread(p, *a))
    got = det.run_images(paths)
    assert read == [paths[-1]]
    for n in range(len(paths)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n
