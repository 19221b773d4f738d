"""GPU tests of the batched raw-image path: cpb200_pre_process_batch, cpb200_soft_nms_39_batch and
MultiPoseDetector.run_images (flip test, multi-scale, FIX_RES, soft-NMS) against run() and the reference's run()."""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

_DET = {}


def _detector(precision="fp16x2", flip=True, nms=True, fix_res=False, scales=(1,)):
    """One conditioned DLA-34 detector per precision; the test section is set per call (run() and run_images read
    cfg.TEST at call time)."""
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    if precision not in _DET:
        cfg = default_cfg("dla_34")
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        det.model.set_precision(precision)
        _DET[precision] = det
    det = _DET[precision]
    det.cfg.TEST.FLIP_TEST = flip
    det.cfg.TEST.NMS = nms
    det.cfg.TEST.FIX_RES = fix_res
    det.cfg.TEST.TEST_SCALES = list(scales)
    det.scales = det.cfg.TEST.TEST_SCALES
    return det


def _images(shapes, seed):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for h, w in shapes]


def _pre_process_batch(det, images, trans, inp_h, inp_w, flip):
    from centerpose_b200 import _lib
    from centerpose_b200.detector import _PRE_IMAGE
    table = np.zeros(len(images), _PRE_IMAGE)
    pos = 0
    for n, (im, t) in enumerate(zip(images, trans)):
        table[n] = (pos, im.shape[0], im.shape[1], np.asarray(t, np.float64).reshape(6))
        pos += im.nbytes
    pix = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
    tab = torch.from_numpy(table.view(np.uint8).copy()).cuda()
    out = torch.full(((2 if flip else 1) * len(images), 3, inp_h, inp_w), float("nan"), device="cuda")
    mean = (ctypes.c_float * 3)(*det.mean.reshape(-1)); std = (ctypes.c_float * 3)(*det.std.reshape(-1))
    _lib.launch("pre_process_batch", out.device, pix, tab, len(images), out, inp_h, inp_w, mean, std, 1 if flip else 0)
    return out


@pytest.mark.parametrize("fix_res", [True, False])
@pytest.mark.parametrize("flip", [False, True])
def test_pre_process_batch_equals_per_image_kernel(fix_res, flip):
    """Every image of one batched launch == cpb200_pre_process on that image alone (torch.equal), mixed image sizes
    sharing one input size, at scale 1 and 0.75 (host cv2.resize first)."""
    det = _detector("fp32", flip=flip, fix_res=fix_res)
    shapes = [(480, 640), (333, 500), (720, 405), (512, 512)] if fix_res else [(240, 320), (250, 330), (225, 340)]
    images = _images(shapes, 21)
    for scale in (1.0, 0.75):
        import cv2
        geo = [det._pre_process_geometry(h, w, scale) for h, w in shapes]
        if not fix_res and scale != 1.0:
            keep = [i for i in range(len(shapes)) if geo[i][2:4] == geo[0][2:4]]
            images_s, geo = [images[i] for i in keep], [geo[i] for i in keep]
            assert len(images_s) >= 2
        else:
            images_s = images
        assert len({g[2:4] for g in geo}) == 1
        resized = [im if (g[1], g[0]) == im.shape[1::-1] else np.ascontiguousarray(cv2.resize(im, (g[1], g[0])))
                   for im, g in zip(images_s, geo)]
        out = _pre_process_batch(det, resized, [g[4] for g in geo], geo[0][2], geo[0][3], flip)
        per = 2 if flip else 1
        for n, im in enumerate(images_s):
            want, _ = det.pre_process(im, scale)
            assert torch.equal(out[per * n:per * (n + 1)], want), (scale, n)
    # and against the host cv2.warpAffine / numpy branch of pre_process (base_detector.py:44-55)
    geo = [det._pre_process_geometry(h, w, 1.0) for h, w in shapes]
    got = _pre_process_batch(det, images, [g[4] for g in geo], geo[0][2], geo[0][3], flip).cpu()
    det.device_preprocess = False
    try:
        for n, im in enumerate(images):
            want, _ = det.pre_process(im, 1.0)
            assert not want.is_cuda and torch.equal(got[per * n:per * (n + 1)], want), n
    finally:
        det.device_preprocess = True


def _nms_rows(rng, B, N):
    rows = np.zeros((B, N, 56), np.float32)
    c = rng.uniform(0, 400, size=(B, N, 2)); wh = rng.uniform(5, 150, size=(B, N, 2))
    rows[..., 0:2] = c - wh / 2; rows[..., 2:4] = c + wh / 2
    rows[..., 4] = rng.uniform(0, 1, (B, N)); rows[..., 5:] = rng.uniform(0, 400, size=(B, N, 51))
    rows[0, :, 4] = np.round(rows[0, :, 4], 1)                       # score ties in one image
    return rows


def _singles(rows, **kw):
    from centerpose_b200.soft_nms import soft_nms_39_cuda
    outs, keeps = [], []
    for r in rows:
        d = torch.from_numpy(r.copy()).cuda()
        keeps.append(soft_nms_39_cuda(d, **kw)); outs.append(d.cpu())
    return torch.stack(outs), keeps


@pytest.mark.parametrize("N", [100, 200])
def test_soft_nms_batch_equals_single_image_calls(N):
    from centerpose_b200.soft_nms import soft_nms_39_cuda_batch
    rows = _nms_rows(np.random.RandomState(N), 5, N)
    for kw in (dict(Nt=0.5, method=2), dict(Nt=0.3, threshold=0.05, method=1), dict(Nt=0.7, method=0)):
        want, keep_want = _singles(rows, **kw)
        dev = torch.from_numpy(rows.copy()).cuda()
        keep = soft_nms_39_cuda_batch(dev, **kw)
        assert keep.dtype == torch.int32 and keep.shape == (5,)
        assert keep.cpu().tolist() == keep_want, kw
        assert torch.equal(dev.cpu(), want), kw
        assert 0 < min(keep_want) < N                                  # suppression happened
    assert soft_nms_39_cuda_batch(torch.zeros(3, 0, 56, device="cuda")).cpu().tolist() == [0, 0, 0]
    with pytest.raises(RuntimeError, match=r"N = 900 rows do not fit shared memory \(max 882\)"):
        soft_nms_39_cuda_batch(torch.zeros(2, 900, 56, device="cuda"))


def test_soft_nms_batch_on_golden_cases():
    """tests/golden/soft_nms.npz (the reference's compiled Cython soft_nms_39): the cases stacked into one batch per
    parameter set equal single-image calls bit for bit, and each case batched at its own N reproduces the golden
    rows and keep count."""
    from centerpose_b200.soft_nms import soft_nms_39_cuda_batch
    g = np.load(os.path.join(GOLD, "soft_nms.npz"))
    groups = {}
    for n, prm in enumerate(g["params"]):
        groups.setdefault((int(prm[1]), float(prm[2]), float(prm[3])), []).append(n)
    for (method, Nt, thr), idx in groups.items():
        kw = dict(sigma=0.5, Nt=Nt, threshold=thr, method=method)
        stacked = g["boxes"][idx]                                     # (len(idx), 100, 56), zero rows beyond each N
        want, keep_want = _singles(stacked, **kw)
        dev = torch.from_numpy(stacked.copy()).cuda()
        assert soft_nms_39_cuda_batch(dev, **kw).cpu().tolist() == keep_want
        assert torch.equal(dev.cpu(), want)
        for n in idx:
            N = int(g["params"][n][0])
            dev = torch.from_numpy(np.repeat(g["boxes"][n][None, :N], 3, axis=0)).cuda()
            assert soft_nms_39_cuda_batch(dev, **kw).cpu().tolist() == [int(g["keep"][n])] * 3
            assert np.abs(dev.cpu().numpy() - g["out"][n][None, :N]).max() <= 2e-7


def _assert_like_run(got, want, what):
    from tests.util import match_rows
    assert got.dtype == np.float32 and got.shape == want.shape, (what, got.shape, want.shape)
    err = float(np.abs(got - want).max())
    assert err <= 2e-3 * max(1.0, float(np.abs(want).max())), (what, err, match_rows(got, want, tol=2e-3, box_tol=5e-2))


@pytest.mark.parametrize("case", ["dla34_test_section", "scales_1_075_flip", "fix_res_no_flip_no_nms"])
def test_run_images_matches_run(case):
    if case == "dla34_test_section":
        det = _detector("fp16x2", flip=True, nms=True, fix_res=False)
        shapes = [(240, 320), (300, 200), (250, 330), (427, 640), (225, 340)]     # 256x352 x3, 320x224, 448x672
    elif case == "scales_1_075_flip":
        det = _detector("fp16x2", flip=True, nms=True, fix_res=False, scales=(1, 0.75))
        shapes = [(240, 320), (300, 200), (250, 330)]
    else:
        det = _detector("fp16x2", flip=False, nms=False, fix_res=True)
        shapes = [(480, 640), (333, 500), (720, 405)]
    images = _images(shapes, 31)
    if case == "dla34_test_section":
        assert len({det._pre_process_geometry(h, w, 1)[2:4] for h, w in shapes}) == 3
    got = det.run_images(images)
    assert len(got) == len(images)
    for n, im in enumerate(images):
        want = np.asarray(det.run(im)["results"][1], dtype=np.float32)
        _assert_like_run(got[n], want, (case, n))


def test_run_images_batch_size_does_not_change_rows(tmp_path):
    import cv2
    det = _detector("fp16x2", flip=True, nms=True, fix_res=False, scales=(1, 0.75))
    images = _images([(240, 320), (300, 200), (250, 330), (225, 340)], 41)
    path = str(tmp_path / "img.png")
    cv2.imwrite(path, images[1])
    a = det.run_images(images)
    b = det.run_images(images, max_batch=1)
    c = det.run_images([images[0], path] + images[2:], max_batch=2)
    for n in range(len(images)):
        assert np.array_equal(a[n], b[n]), n
        assert np.array_equal(a[n], c[n]), n


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
def test_run_images_matches_reference_run_fixture(precision):
    """tests/golden/run_dla34_flip.npz: the reference's own run() on the CPU (oracle/make_golden_run.py)."""
    from oracle import make_golden_run as g
    from tests.util import match_rows
    f = np.load(os.path.join(GOLD, "run_dla34_flip.npz"))
    images = g.make_images()
    assert str(f["img_sha"]) == g._sha(*images)
    report = []
    for case, scales in g.CASES.items():
        det = _detector(precision, flip=True, nms=True, fix_res=False, scales=scales)
        got = det.run_images(images)
        for n in range(len(images)):
            want = f[f"rows_{case}_{n}"]
            assert got[n].shape == want.shape
            rows, elems = match_rows(got[n], want, tol=2e-3, box_tol=5e-2)
            report.append((case, n, round(rows, 4), round(elems, 4)))
            assert rows >= 0.9 and elems >= 0.97, (precision, case, n, rows, elems)
    print(precision, "run_images vs reference run():", report)


def test_run_multiscale_fused_supports_flip():
    det = _detector("fp16x2", flip=True, nms=False, fix_res=False, scales=(1, 0.75))
    image = _images([(384, 512)], 11)[0]
    want = np.asarray(det.run(image)["results"][1], dtype=np.float32)
    _assert_like_run(det.run_multiscale_fused(image), want, "run_multiscale_fused")


def test_run_images_rejects_bad_input():
    det = _detector("fp16x2", flip=False, nms=False, fix_res=True)
    good = _images([(64, 64)], 1)[0]
    assert det.run_images([]) == []
    for bad in (good.astype(np.float32), good[:, :, :2], good[:, :, 0], np.zeros((8, 8, 4), np.uint8), 7, None):
        with pytest.raises(ValueError):
            det.run_images([good, bad])
    with pytest.raises(ValueError):
        det.run_images([good], max_batch=0)
