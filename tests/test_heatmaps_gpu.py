"""GPU tests of the heat-map views (cpb200_heatmap_views_batch): the kernels against the reference Debugger's golden
views and the numpy / cv2 oracle byte for byte, run() with DEBUG 2, and run_images(..., return_heatmaps=True)."""
import os

import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import heatmaps
from oracle import debugger_ref, heatmaps_ref
from tests import render_cases as rc
from tests.test_heatmaps_cpu import THEMES, golden_cases

pytestmark = pytest.mark.gpu

_DET = {}
MIXED = [(512, 512), (480, 640), (640, 480), (992, 1312), (32, 160), (4, 4)]


def _detector(theme="white", flip=False, scales=(1,), mse=False):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    if "det" not in _DET:
        cfg = default_cfg("dla_34")
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        _DET["det"] = det
    det = _DET["det"]
    det.cfg.DEBUG_THEME = theme
    det.cfg.DEBUG = 0
    det.cfg.TEST.VIS_THRESH = 0.05
    det.cfg.TEST.FLIP_TEST = flip
    det.cfg.TEST.TEST_SCALES = list(scales)
    det.scales = det.cfg.TEST.TEST_SCALES
    det.cfg.LOSS.MSE_LOSS = mse
    return det


def mixed_inputs(seed=5):
    """Inputs for MIXED: de-normalized values uniform over [-8, 263] (every back byte, clipped ones included), hm maps
    that make every colour-map byte, keypoint maps with NaN, negative and out-of-range values."""
    rng = np.random.default_rng(seed)
    mean, std = np.array([0.408, 0.447, 0.470], np.float32), np.array([0.289, 0.274, 0.278], np.float32)
    out = []
    for H, W in MIXED:
        h, w = H // 4, W // 4
        b = rng.uniform(-8, 263, (3, H, W)).astype(np.float32)
        x = ((b / 255 - mean.reshape(3, 1, 1)) / std.reshape(3, 1, 1)).astype(np.float32)
        # 2x2 blocks of one value, so the colour map has runs of every byte the resizes keep
        k = rng.integers(0, 256, (1, (h + 1) // 2, (w + 1) // 2)).repeat(2, 1).repeat(2, 2)[:, :h, :w]
        hm = np.minimum((k + 0.5) / 255, 1).astype(np.float32)
        hp = rng.random((17, h, w)).astype(np.float32) ** 3
        hp.reshape(-1)[:4] = [np.nan, -0.5, 1.7, 3e9]
        out.append((x, hm, hp))
    return out, mean, std


def _views(inputs, theme, mean, std, dr=4):
    dev = [tuple(torch.from_numpy(a).cuda() for a in t) for t in inputs]
    return heatmaps.views([d[0] for d in dev], [d[1] for d in dev], [d[2] for d in dev], dr, theme, mean, std)


def test_views_equal_golden():
    cases, mean, std = golden_cases()
    for theme in THEMES:
        for dr in sorted({c[3] for c in cases}):
            sel = [c for c in cases if c[3] == dr]
            got = _views([c[:3] for c in sel], theme, mean, std, dr)
            for (x, hm, hp, _, want), g in zip(sel, got):
                for v in heatmaps.VIEWS:
                    assert g[v].dtype == np.uint8 and g[v].shape == x.shape[1:] + (3,)
                    assert np.array_equal(g[v], want[theme][v]), (theme, hp.shape, v)


@pytest.mark.parametrize("theme", THEMES)
def test_mixed_sizes_in_one_call_equal_oracle(theme):
    inputs, mean, std = mixed_inputs()
    got = _views(inputs, theme, mean, std)
    pairs = np.zeros(65536, bool)
    hm_color, hp_colors = heatmaps_ref.map_colors(theme)
    for (x, hm, hp), g in zip(inputs, got):
        want = heatmaps_ref.heatmap_views(x, hm, hp, 4, theme, mean, std)
        for v in heatmaps.VIEWS:
            assert np.array_equal(g[v], want[v]), (x.shape, v, np.argwhere(g[v] != want[v])[:5].tolist())
        back = heatmaps_ref.back_image(x, mean, std).astype(np.int64)
        fore = heatmaps_ref.fore_image(hm, hm_color, 4, theme, *x.shape[1:]).astype(np.int64)
        pairs[(back * 256 + fore).reshape(-1)] = True
    assert pairs.all(), "the blend saw %d of the 65536 (back, fore) pairs" % pairs.sum()


def _spy(det):
    """Records each debug() call's input and maps as numpy arrays."""
    calls = []
    orig = type(det).debug

    def debug(debugger, images, dets, output, scale=1):
        calls.append((images[0].cpu().numpy(), output[0][0].cpu().numpy(), output[4][0].cpu().numpy()))
        return orig(det, debugger, images, dets, output, scale)
    det.debug = debug
    return calls


@pytest.mark.parametrize("flip,scales,mse,theme", [(False, (1,), False, "white"), (True, (1,), False, "black"),
                                                   (False, (1, 2), False, "black"), (True, (1, 0.75), True, "white"),
                                                   (False, (1,), True, "black")])
def test_run_debug_2(flip, scales, mse, theme):
    det = _detector(theme, flip, scales, mse)
    img = rc.image(240, 320, 11)
    plain = det.run(img)["results"][1]
    calls = _spy(det)
    det.cfg.DEBUG = 2
    try:
        out = det.run(img)
    finally:
        det.cfg.DEBUG = 0
        del det.debug
        det.cfg.LOSS.MSE_LOSS = False
    assert out["results"][1] == plain
    assert len(calls) == len(scales) and list(det.debug_imgs) == ["pred_hm", "pred_hmhp", "multi_pose"]
    x, hm, hp = calls[-1]
    if mse:
        assert (hp < 0).any() and not ((hm < 0) | (hm > 1)).any()
    else:
        assert not ((hp < 0) | (hp > 1)).any()
    want = heatmaps_ref.heatmap_views(x, hm, hp, 4, theme, det.mean, det.std)
    for v in heatmaps.VIEWS:
        assert np.array_equal(det.debug_imgs[v], want[v]), v
        assert det.debug_imgs[v].shape == x.shape[1:] + (3,)
    assert np.array_equal(det.debug_imgs["multi_pose"], debugger_ref.show_results(img, out["results"][1], 0.05, theme))
    det.cfg.DEBUG = 1
    try:
        det.run(img)
    finally:
        det.cfg.DEBUG = 0
    assert list(det.debug_imgs) == ["multi_pose"]


def _write_jpegs(tmp_path, n):
    paths = []
    for k in range(n):
        h, w = [(480, 640), (640, 480), (427, 640), (333, 501)][k % 4]
        p = os.path.join(str(tmp_path), "im%d.jpg" % k)
        cv2.imwrite(p, rc.image(h, w, 500 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    return paths


@pytest.mark.parametrize("source,flip,images", [("jpeg", False, False), ("arrays", False, True), ("jpeg", True, True),
                                                ("arrays", True, False)])
def test_run_images_return_heatmaps(tmp_path, source, flip, images):
    det = _detector("white", flip, (1, 0.75) if flip else (1,))
    paths = _write_jpegs(tmp_path, 5)
    inputs = paths if source == "jpeg" else [cv2.imread(p) for p in paths]
    plain = det.run_images(inputs, max_batch=2)
    res = det.run_images(inputs, max_batch=2, return_images=images, return_heatmaps=True)
    assert len(res) == (3 if images else 2)
    rows, views = res[0], res[-1]
    assert len(rows) == len(views) == len(inputs)
    calls = _spy(det)
    det.cfg.DEBUG = 2
    try:
        for n, (p, r, vw, src) in enumerate(zip(plain, rows, views, inputs)):
            assert np.array_equal(p, r)
            det.run(src)
            for v in heatmaps.VIEWS:
                assert np.array_equal(vw[v], det.debug_imgs[v]), (n, v)
            x, hm, hp = calls[-1]
            assert vw["pred_hm"].shape == x.shape[1:] + (3,)
            if images:
                img = cv2.imread(paths[n])
                assert np.array_equal(res[1][n], debugger_ref.show_results(img, r.tolist(), 0.05, "white"))
    finally:
        det.cfg.DEBUG = 0
        del det.debug
    assert det.run_images([], return_heatmaps=True) == ([], [])
    assert det.run_images([], return_images=True, return_heatmaps=True) == ([], [], [])
