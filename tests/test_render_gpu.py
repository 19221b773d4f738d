"""GPU tests of the pose drawing (cpb200_render_poses_batch): render_poses, run_images(..., return_images=True) and
run() with DEBUG 1 against the reference Debugger's golden images and the cv2 oracle, byte for byte."""
import os

import cv2
import numpy as np
import pytest

from oracle import debugger_ref
from tests import render_cases as rc
from tests.test_render_cpu import golden_cases

pytestmark = pytest.mark.gpu

_DET = {}


def _detector(theme="white", vis_thresh=0.3):
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
    det.cfg.TEST.VIS_THRESH = vis_thresh
    det.cfg.DEBUG = 0
    return det


def test_render_poses_equals_golden():
    cases = golden_cases()
    for theme in ("white", "black"):
        sel = [c for c in cases if c[2] == theme]
        got = _detector(theme).render_poses([c[0] for c in sel], [c[1] for c in sel])
        for (img, rows, _, out), g in zip(sel, got):
            assert g.dtype == np.uint8 and g.shape == img.shape
            assert np.array_equal(g, out)


@pytest.mark.parametrize("theme", ["white", "black"])
def test_render_poses_mixed_sizes_equals_oracle(theme):
    shapes = [(480, 640), (640, 480), (427, 640), (992, 1312), (31, 17), (1, 1), (700, 99), (99, 701), (3, 900)]
    images = [rc.image(h, w, 50 + k) for k, (h, w) in enumerate(shapes)]
    results = []
    for k, (h, w) in enumerate(shapes):
        n = [5, 10, 1, 100, 7, 3, 30, 20, 4][k]
        r = rc.rows(h, w, n, 60 + k, spread=0.5, off=0.25)
        r[:, 4] = np.where(np.arange(n) % 5 == 4, r[:, 4], 0.31 + 0.68 * np.random.default_rng(k).random(n))
        if k == 4:
            r = np.concatenate([r, rc.edge_rows(h, w)])
        results.append(r)
    results[5] = results[5][:0]                                        # no rows at all
    det = _detector(theme)
    got = det.render_poses(images, results)
    assert sum(int((r[:, 4].astype(np.float64) > 0.3).sum()) for r in results) > 150
    for img, rows, g in zip(images, results, got):
        want = debugger_ref.show_results(img, rows.tolist(), 0.3, theme)
        assert np.array_equal(g, want), (img.shape, np.argwhere((g != want).any(2))[:5].tolist())
    for img, g in zip(images, det.render_poses(images, results)):     # the input images are not drawn on
        assert not np.shares_memory(img, g)


def _write_jpegs(tmp_path, n):
    paths = []
    for k in range(n):
        h, w = [(480, 640), (640, 480), (427, 640), (333, 501)][k % 4]
        p = os.path.join(str(tmp_path), "im%d.jpg" % k)
        cv2.imwrite(p, rc.image(h, w, 400 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])
        paths.append(p)
    return paths


@pytest.mark.parametrize("source", ["jpeg", "arrays"])
def test_run_images_return_images(tmp_path, source):
    det = _detector("white", vis_thresh=0.05)
    paths = _write_jpegs(tmp_path, 6)
    inputs = paths if source == "jpeg" else [cv2.imread(p) for p in paths]
    plain = det.run_images(inputs)
    rows, drawn = det.run_images(inputs, return_images=True)
    assert len(rows) == len(plain) == len(drawn)
    n_drawn = 0
    for p, r, d, src in zip(plain, rows, drawn, inputs):
        assert np.array_equal(p, r)
        img = cv2.imread(src) if isinstance(src, str) else src
        n_drawn += int((r[:, 4].astype(np.float64) > 0.05).sum())
        assert np.array_equal(d, debugger_ref.show_results(img, r.tolist(), 0.05, "white"))
    assert n_drawn > 0
    assert det.run_images([], return_images=True) == ([], [])


def test_run_debug_1_fills_debug_imgs():
    det = _detector("black", vis_thresh=0.05)
    det.cfg.DEBUG = 1
    img = rc.image(240, 320, 7)
    try:
        out = det.run(img)
    finally:
        det.cfg.DEBUG = 0
    want = debugger_ref.show_results(img, out["results"][1], 0.05, "black")
    assert np.array_equal(det.debug_imgs["multi_pose"], want)
    assert not np.array_equal(want, img)
