"""GPU tests of the device resize: cpb200_resize_linear_u8_batch against cv2.resize, and pre_process / run_images at
test scales != 1 against the host cv2 path (``DEVICE_PREPROCESS: false``)."""
import numpy as np
import pytest
import torch

from tests.test_resize_cpu import SCALES, SIZES

pytestmark = pytest.mark.gpu
CPB200_ERR_ARG = 1


def _launch(src, table, B, dst):
    from centerpose_b200 import _lib
    return _lib.lib().cpb200_resize_linear_u8_batch(src, table, B, dst, torch.cuda.current_stream().cuda_stream)


def _resize_batch(images, new_shapes):
    """One launch over all images; returns the resized images (numpy) after checking the bytes behind the last one
    were left alone."""
    from centerpose_b200 import _lib
    from centerpose_b200.detector import resize_table
    table = resize_table([im.shape[0:2] for im in images], new_shapes)
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    total = sum(h * w * 3 for h, w in new_shapes)
    dst = torch.full((total + 256,), 77, dtype=torch.uint8, device="cuda")
    _lib.check(_launch(src.data_ptr(), tab.data_ptr(), len(images), dst.data_ptr()), "resize_linear_u8_batch")
    out = dst.cpu().numpy()
    assert (out[total:] == 77).all()
    return [out[e["dst_offset"]:e["dst_offset"] + e["new_h"] * e["new_w"] * 3].reshape(e["new_h"], e["new_w"], 3)
            for e in table]


def _grid_images(seed):
    rng = np.random.RandomState(seed)
    images, new_shapes = [], []
    for (h, w) in SIZES:
        for scale in SCALES:
            if int(h * scale) >= 1 and int(w * scale) >= 1:
                images.append(rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
                new_shapes.append((int(h * scale), int(w * scale)))
    return images, new_shapes


def test_resize_kernel_equals_cv2_on_the_grid():
    """Every (size, scale) of the CPU grid: once per scale (mixed sizes in one launch) and all of them in one launch,
    byte for byte against cv2.resize."""
    import cv2
    images, new_shapes = _grid_images(3)
    for scale in SCALES:
        idx = [n for n, (im, s) in enumerate(zip(images, new_shapes)) if s == (int(im.shape[0] * scale), int(im.shape[1] * scale))]
        got = _resize_batch([images[n] for n in idx], [new_shapes[n] for n in idx])
        for n, g in zip(idx, got):
            want = cv2.resize(images[n], new_shapes[n][::-1])
            assert np.array_equal(g, want), (images[n].shape, new_shapes[n], int((g != want).sum()))
    got = _resize_batch(images, new_shapes)
    for im, s, g in zip(images, new_shapes, got):
        assert np.array_equal(g, cv2.resize(im, s[::-1])), (im.shape, s)


def test_resize_batched_equals_single_image_calls():
    images, new_shapes = _grid_images(4)
    rng = np.random.RandomState(4)
    images += [rng.randint(0, 256, (480, 640, 3)).astype(np.uint8), rng.randint(0, 256, (427, 640, 3)).astype(np.uint8)]
    new_shapes += [(960, 1280), (320, 480)]
    batched = _resize_batch(images, new_shapes)
    for im, s, b in zip(images, new_shapes, batched):
        assert np.array_equal(_resize_batch([im], [s])[0], b), (im.shape, s)


def test_resize_rejects_host_checkable_arguments():
    """B < 1, B > 65535 and null pointers return CPB200_ERR_ARG without a launch; the kernel only ever sees a valid
    device table."""
    from centerpose_b200 import _lib
    from centerpose_b200.detector import resize_table
    table = resize_table([(4, 6)], [(8, 12)])
    src = torch.zeros(4 * 6 * 3, dtype=torch.uint8, device="cuda")
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    dst = torch.full((8 * 12 * 3,), 77, dtype=torch.uint8, device="cuda")
    s, t, d = src.data_ptr(), tab.data_ptr(), dst.data_ptr()
    for args in ((s, t, 0, d), (s, t, -1, d), (s, t, 65536, d), (None, t, 1, d), (s, None, 1, d), (s, t, 1, None)):
        assert _launch(*args) == CPB200_ERR_ARG, args
        assert b"resize_linear_u8_batch" in _lib.lib().cpb200_last_error()
    torch.cuda.synchronize()
    assert (dst.cpu().numpy() == 77).all()
    assert _launch(s, t, 1, d) == 0
    assert (dst.cpu().numpy() == 0).all()


_DET = {}


def _detector(arch, precision, scales, flip):
    """Conditioned weights; the test section of experiments/{dla_34_512x512,hrnet_w32_512}.yaml (FIX_RES false,
    soft-NMS through the multi-scale merge) with the given scales and flip."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from centerpose_b200.synth import conditioned_state_dict
    if (arch, precision) not in _DET:
        cfg = default_cfg(arch)
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        det.model.set_precision(precision)
        _DET[(arch, precision)] = det
    det = _DET[(arch, precision)]
    det.cfg.TEST.FLIP_TEST = flip
    det.cfg.TEST.NMS = arch == "dla_34"
    det.cfg.TEST.FIX_RES = False
    det.cfg.TEST.TEST_SCALES = list(scales)
    det.scales = det.cfg.TEST.TEST_SCALES
    det.device_preprocess = True
    return det


def _host_run(det, image):
    det.device_preprocess = False
    try:
        return np.asarray(det.run(image)["results"][1], dtype=np.float32)
    finally:
        det.device_preprocess = True


@pytest.mark.parametrize("scale", [2, 0.75, 1.25])
@pytest.mark.parametrize("flip", [False, True])
def test_pre_process_device_resize_equals_host_cv2(scale, flip):
    """The network input of pre_process at a scale != 1 is the same tensor with the device resize as with cv2."""
    det = _detector("dla_34", "fp32", (1, scale), flip)
    rng = np.random.RandomState(8)
    for h, w in [(120, 160), (333, 500), (37, 51), (1, 9)]:
        image = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        if int(h * scale) < 1:
            with pytest.raises(ValueError):
                det.pre_process(image, scale)
            continue
        got, meta = det.pre_process(image, scale)
        det.device_preprocess = False
        want, meta_h = det.pre_process(image, scale)
        det.device_preprocess = True
        assert got.is_cuda and not want.is_cuda and torch.equal(got.cpu(), want), (h, w)
        assert all(np.array_equal(meta[k], meta_h[k]) for k in meta)


RUN_CASES = [("dla_34", p, s, f) for p in ("fp32", "fp16x2") for s in ((1, 2), (1, 0.75)) for f in (True, False)]
RUN_CASES += [("hrnet", "fp16x2", (1, 2), True)]                       # experiments/hrnet_w32_512.yaml, TEST section


@pytest.mark.parametrize("arch,precision,scales,flip", RUN_CASES)
def test_run_images_multiscale_equals_host_cv2_run(arch, precision, scales, flip):
    """run() with the device resize returns the same floats as run() with the host cv2.resize: the network inputs are
    the same bits and everything after them is the same code.  run_images (raw pixels uploaded, batched device resize)
    agrees with them up to the fused back-projection: the decode applies the float32 matrix divided by the scale, where
    post_process applies the float64 one and divides afterwards.  At scale 2 the two differ only where the float64
    matrix is not exactly representable (the 100x150 image: a -1.8e-16 entry), at 0.75 wherever 1/0.75 rounds; by an
    ulp or two of the coordinates either way, far inside the 2e-3 of tests/test_run_images_gpu.py."""
    det = _detector(arch, precision, scales, flip)
    shapes = [(120, 160), (100, 150), (130, 170), (120, 160)] if arch == "dla_34" else [(120, 160), (100, 150)]
    rng = np.random.RandomState(51)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    got = det.run_images(images, max_batch=32 if arch == "dla_34" else 1)
    for n, im in enumerate(images):
        want = _host_run(det, im)
        assert np.array_equal(np.asarray(det.run(im)["results"][1], dtype=np.float32), want), n
        assert got[n].dtype == np.float32 and got[n].shape == want.shape == (100 * len(scales), 56)
        err = float(np.abs(got[n] - want).max())
        print(arch, precision, scales, flip, "image", n, "run_images vs run() max |diff|", err)
        assert err <= 1e-6 * max(1.0, float(np.abs(want).max())), (n, err)
