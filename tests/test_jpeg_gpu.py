"""GPU tests of the device JPEG decoder: cpb200_jpeg_decode_batch against cv2.imdecode / cv2.imread, its status on bad
entropy data, and MultiPoseDetector.run_images on paths against run_images on the cv2.imread arrays."""
import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import jpeg
from tests.test_jpeg_cpu import CONTENTS, QUALITIES, SAMPLINGS, SIZES, cv2_decode, encode, make_image, with_exif

pytestmark = pytest.mark.gpu
CPB200_ERR_ARG = 1
COCO = [(480, 640), (640, 480), (427, 640)]


def _launch(src, table, B, ws, ws_bytes, dst, status):
    from centerpose_b200 import _lib
    return _lib.lib().cpb200_jpeg_decode_batch(src, table, B, ws, ws_bytes, dst, status,
                                               torch.cuda.current_stream().cuda_stream)


def _decode(datas):
    """One launch over all files; returns (images, status) after checking the bytes behind the last image were left
    alone."""
    from centerpose_b200 import _lib
    infos = [jpeg.parse(d) for d in datas]
    assert all(i.eligible for i in infos)
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = jpeg.pack(infos, datas, offs[:-1])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
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
                    for rst in (0, 3):
                        im = make_image(h, w, content, h * 7 + w + quality, gray=gray)
                        files.append(encode(im, quality, sampling, rst=rst))
        for quality in (75, 95):
            for h, w in COCO:
                for content in CONTENTS:
                    files.append(encode(make_image(h, w, content, h + w + quality, gray=gray), quality, sampling))
    return files


def test_jpeg_kernel_equals_cv2_imdecode():
    """The CPU grid (sizes 1x1 to 97x131, qualities 10-100, 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 / grayscale, with and
    without restart markers, three contents) plus COCO-sized images, mixed in one launch, byte for byte."""
    files = _grid_files()
    got, status = _decode(files)
    assert (status == 0).all()
    bad = [n for n, (g, d) in enumerate(zip(got, files)) if not np.array_equal(g, cv2_decode(d))]
    assert not bad, (len(bad), bad[:10])


def test_jpeg_batched_equals_single_image_calls():
    files = _grid_files()[::17]
    batched, _ = _decode(files)
    for d, b in zip(files, batched):
        single, status = _decode([d])
        assert status[0] == 0 and np.array_equal(single[0], b)


@pytest.mark.parametrize("sampling", ["420", "444", "gray"])
def test_jpeg_exif_orientation_equals_cv2_imread(tmp_path, sampling):
    files = []
    for o in range(1, 9):
        data = with_exif(encode(make_image(37, 61, "smooth_noise", o, gray=sampling == "gray"), 85, sampling), o)
        files.append(data)
    got, status = _decode(files)
    assert (status == 0).all()
    for o, (d, g) in enumerate(zip(files, got), 1):
        path = str(tmp_path / ("o%d.jpg" % o))
        with open(path, "wb") as f:
            f.write(d)
        want = cv2.imread(path)
        assert g.shape == want.shape == ((61, 37, 3) if o >= 5 else (37, 61, 3)), o
        assert np.array_equal(g, want), o


def _truncated():
    data = encode(make_image(96, 128, "noise", 9), 95, "420")
    return data[:len(data) * 2 // 3]


def test_jpeg_bad_entropy_data_sets_status_and_spares_neighbours():
    good = [encode(make_image(64, 80, c, 3), 90, s) for c in CONTENTS for s in ("420", "444")]
    files = good[:3] + [_truncated()] + good[3:]
    got, status = _decode(files)
    assert status.tolist() == [0, 0, 0, 1, 0, 0, 0]
    for n, (d, g) in enumerate(zip(files, got)):
        if n != 3:
            assert np.array_equal(g, cv2_decode(d)), n


def test_jpeg_rejects_host_checkable_arguments():
    from centerpose_b200 import _lib
    data = encode(make_image(16, 16, "noise", 1), 75, "420")
    info = jpeg.parse(data)
    buf, ws_bytes = jpeg.pack([info], [data], [0])
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.full((16 * 16 * 3,), 77, dtype=torch.uint8, device="cuda")
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    s, w, d, st = src.data_ptr(), ws.data_ptr(), dst.data_ptr(), status.data_ptr()
    for args in ((s, s, 0, w, ws_bytes, d, st), (s, s, -1, w, ws_bytes, d, st), (s, s, 65536, w, ws_bytes, d, st),
                 (None, s, 1, w, ws_bytes, d, st), (s, None, 1, w, ws_bytes, d, st), (s, s, 1, None, ws_bytes, d, st),
                 (s, s, 1, w, ws_bytes, None, st), (s, s, 1, w, ws_bytes, d, None)):
        assert _launch(*args) == CPB200_ERR_ARG, args
        assert b"jpeg_decode_batch" in _lib.lib().cpb200_last_error()
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 77).all() and status.item() == -1
    # a workspace too small for the image: status 2, nothing decoded
    assert _launch(s, s, 1, w, ws_bytes - 1, d, st) == 0
    assert status.item() == 2 and (dst.cpu().numpy() == 77).all()
    assert _launch(s, s, 1, w, ws_bytes, d, st) == 0
    assert status.item() == 0 and np.array_equal(dst.cpu().numpy().reshape(16, 16, 3), cv2_decode(data))


_DET = {}


def _detector(arch, precision, scales):
    """Conditioned weights and the test section of experiments/{dla_34_512x512,hrnet_w32_512}.yaml, with ``scales``."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from centerpose_b200.synth import conditioned_state_dict
    if (arch, precision) not in _DET:
        cfg = default_cfg(arch)
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        det.model.set_precision(precision)
        _DET[(arch, precision)] = (det, list(cfg.TEST.TEST_SCALES))
    det, default_scales = _DET[(arch, precision)]
    det.cfg.TEST.TEST_SCALES = list(scales) if scales else default_scales
    det.scales = det.cfg.TEST.TEST_SCALES
    det.device_preprocess = True
    return det


def _files(tmp_path, specs):
    paths = []
    for n, (h, w, sampling, kw) in enumerate(specs):
        im = make_image(h, w, CONTENTS[n % 3], 100 + n)
        kw = dict(kw)
        orientation = kw.pop("orientation", 0)
        data = encode(im, 90, sampling, **kw)
        if orientation:
            data = with_exif(data, orientation)
        p = str(tmp_path / ("f%d.jpg" % n))
        with open(p, "wb") as f:
            f.write(data)
        paths.append(p)
    return paths


SPECS = [(120, 160, "420", {}), (100, 150, "444", {}), (120, 160, "422", {"rst": 4}), (130, 170, "440", {}),
         (160, 120, "420", {"orientation": 6})]
HOST_SPECS = [(120, 160, "420", {"progressive": True}), (100, 150, "411", {})]
RUN_CASES = [("dla_34", p, s) for p in ("fp32", "fp16x2") for s in (None, (1, 0.75))] + [("hrnet", "fp16x2", None)]


@pytest.mark.parametrize("arch,precision,scales", RUN_CASES)
def test_run_images_paths_equal_run_images_arrays(tmp_path, arch, precision, scales):
    """The same float rows from paths (decoded on the device) as from the cv2.imread arrays, with a progressive and a
    4:1:1 file (host path) mixed in."""
    det = _detector(arch, precision, scales)
    specs = SPECS + HOST_SPECS if arch == "dla_34" else SPECS[:2] + HOST_SPECS[:1]
    paths = _files(tmp_path, specs)
    got = det.run_images(paths, max_batch=32 if arch == "dla_34" else 2)
    want = det.run_images([cv2.imread(p) for p in paths], max_batch=32 if arch == "dla_34" else 2)
    for n in range(len(paths)):
        assert got[n].dtype == np.float32 and np.array_equal(got[n], want[n]), n


def test_run_images_mixed_inputs_truncated_file_and_host_decode(tmp_path):
    """Arrays and paths in one call, a file cut inside its entropy data (device status -> cv2.imread), and
    DEVICE_PREPROCESS false (every path through cv2.imread): all give the rows of the cv2.imread arrays."""
    det = _detector("dla_34", "fp16x2", None)
    paths = _files(tmp_path, SPECS[:3])
    cut = str(tmp_path / "cut.jpg")
    with open(cut, "wb") as f:
        f.write(_truncated())
    assert jpeg.parse(open(cut, "rb").read()).eligible
    arrays = [make_image(110, 140, "noise", 5), make_image(90, 200, "smooth", 6)]
    inputs = [paths[0], arrays[0], cut, paths[1], arrays[1], paths[2]]
    want = det.run_images([cv2.imread(x) if isinstance(x, str) else x for x in inputs])
    got = det.run_images(inputs)
    det.device_preprocess = False
    host = det.run_images(inputs)
    det.device_preprocess = True
    for n in range(len(inputs)):
        assert np.array_equal(got[n], want[n]), n
        assert np.array_equal(host[n], want[n]), n
    with pytest.raises(FileNotFoundError):
        det.run_images([paths[0], str(tmp_path / "missing.jpg")])
