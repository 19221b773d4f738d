"""MultiPoseDetector.run_video on the device: on videos written here (``mp4v`` .mp4) and on iterables, the rows of each
frame equal ``run_images`` on the frames the capture loop reads, bit for bit (the same kernels and tables), and match
``run(frame)`` as ``run_images`` does; the drawn frames equal ``render_poses`` and the reference's Debugger byte for
byte, and their PNG files ``cv2.imencode``.  Under the dla_34 test section and under flip, scales [1, 0.75] with NMS,
in fp32 and fp16x2, at 640x480, 480x640, 1280x720 and 641x359, for 1, max_batch - 1 and max_batch + 1 frames and for a
mixed-shape iterable.  The device drawing plan (``render.DevicePlan``, ``cpb200_render_plan_batch``) draws constructed
rows byte for byte as ``render_poses``: many persons, labels cut by each border, zero-length and off-image limbs,
scores at the threshold, and tables that outgrow their first share; its polygons (``cpb200_ellipse_poly_batch``)
equal tests/ellipse_model.py, and so cv2.ellipse2Poly, over the model's exhaustive domain.  Also: the same results
under a side stream, and the early errors."""
import cv2
import numpy as np
import pytest
import torch

from oracle import debugger_ref
from tests import render_cases as rc
from tests.test_video_cpu import capture_frames, reader_threads

pytestmark = pytest.mark.gpu

MAX_BATCH = 4
SECTIONS = {"dla_34": {"FLIP_TEST": True, "NMS": True, "FIX_RES": False, "TEST_SCALES": [1]},
            "flip_scales_nms": {"FLIP_TEST": True, "NMS": True, "FIX_RES": False, "TEST_SCALES": [1, 0.75]},
            "fix_res": {"FLIP_TEST": False, "NMS": False, "FIX_RES": True, "TEST_SCALES": [1]}}
_DET = {}


def _detector(precision, section):
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from centerpose_b200.synth import conditioned_state_dict
    if precision not in _DET:
        cfg = default_cfg("dla_34")
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        det.model.set_precision(precision)
        _DET[precision] = det
    det = _DET[precision]
    for k, v in SECTIONS[section].items():
        setattr(det.cfg.TEST, k, list(v) if isinstance(v, list) else v)
    det.scales = det.cfg.TEST.TEST_SCALES
    det.cfg.TEST.VIS_THRESH = 0.05            # conditioned weights score low: draw many persons
    return det


def _video(tmp_path, n, h, w, seed=0):
    vw = cv2.VideoWriter(str(tmp_path / ("v%d_%dx%d.mp4" % (n, w, h))), cv2.VideoWriter_fourcc(*"mp4v"), 25, (w, h))
    assert vw.isOpened()
    for i in range(n):
        vw.write(rc.image(h, w, seed + i))
    vw.release()
    return str(tmp_path / ("v%d_%dx%d.mp4" % (n, w, h)))


def _check(det, source, frames, return_images=False, max_batch=MAX_BATCH):
    got = list(det.run_video(source, max_batch=max_batch, return_images=return_images))
    assert [g[0] for g in got] == list(range(len(frames)))
    want = det.run_images(frames, max_batch=max_batch)
    for (i, rows, *drawn), w in zip(got, want):
        assert rows.dtype == np.float32 and np.array_equal(rows, w), i
    assert not reader_threads()
    return got


@pytest.mark.parametrize("precision", ["fp32", "fp16x2"])
@pytest.mark.parametrize("section", ["dla_34", "flip_scales_nms"])
@pytest.mark.parametrize("h,w", [(480, 640), (640, 480), (720, 1280), (359, 641)])
def test_rows_equal_run_images(tmp_path, precision, section, h, w):
    det = _detector(precision, section)
    path = _video(tmp_path, MAX_BATCH + 1, h, w)
    frames = capture_frames(path)
    assert len(frames) == MAX_BATCH + 1
    _check(det, path, frames)


@pytest.mark.parametrize("n", [1, MAX_BATCH - 1, MAX_BATCH + 1])
def test_frame_counts(tmp_path, n):
    det = _detector("fp16x2", "flip_scales_nms")
    path = _video(tmp_path, n, 480, 640, seed=10)
    frames = capture_frames(path)
    assert len(frames) == n
    _check(det, path, frames)


def test_rows_match_run(tmp_path):
    """run() decodes on the host (post_process), so its rows match run_images', and run_video's, within the bound
    tests/test_detector_gpu.py holds run_images to."""
    from tests.util import match_rows
    det = _detector("fp16x2", "flip_scales_nms")
    path = _video(tmp_path, 3, 359, 641, seed=20)
    for (i, rows), frame in zip(det.run_video(path, max_batch=2), capture_frames(path)):
        want = np.asarray(det.run(frame)["results"][1], dtype=np.float32)
        assert abs(len(rows) - len(want)) <= 2
        matched, elems = match_rows(rows, want, tol=2e-3, box_tol=5e-2)
        assert matched >= 0.97 and elems >= 0.99, (i, matched, elems)


@pytest.mark.parametrize("section", ["dla_34", "fix_res"])
def test_mixed_shape_iterable(section):
    det = _detector("fp16x2", section)
    shapes = [(480, 640)] * 2 + [(359, 641)] + [(480, 640)] * 3 + [(640, 480)] * 2
    frames = [rc.image(h, w, 40 + k) for k, (h, w) in enumerate(shapes)]
    _check(det, iter(frames), frames, max_batch=2)


@pytest.mark.parametrize("theme", ["white", "black"])
def test_drawn_frames_equal_render_poses(tmp_path, theme):
    det = _detector("fp16x2", "dla_34")
    det.cfg.DEBUG_THEME = theme
    try:
        path = _video(tmp_path, MAX_BATCH + 2, 359, 641, seed=30)
        frames = capture_frames(path)
        got = _check(det, path, frames, return_images=True)
        for k, ((i, rows, drawn), frame) in enumerate(zip(got, frames)):
            assert np.array_equal(drawn, det.render_poses([frame], [rows])[0]), i
            if k < 2:
                assert np.array_equal(drawn, debugger_ref.show_results(frame, rows.tolist(), 0.05, theme)), i
        pngs = list(det.run_video(path, max_batch=MAX_BATCH, return_images=True, encode_png=True))
        for (i, rows, drawn), (_, rows2, data) in zip(got, pngs):
            assert np.array_equal(rows, rows2)
            assert data == cv2.imencode(".png", drawn)[1].tobytes(), i
    finally:
        det.cfg.DEBUG_THEME = "white"


def test_same_results_on_a_side_stream(tmp_path):
    det = _detector("fp16x2", "flip_scales_nms")
    path = _video(tmp_path, 5, 480, 640, seed=50)

    def fn():
        return list(det.run_video(path, max_batch=2, return_images=True))
    want = fn()
    torch.cuda.synchronize()
    with torch.cuda.stream(torch.cuda.Stream()):
        got = fn()
    torch.cuda.synchronize()
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g[0] == w[0] and np.array_equal(g[1], w[1]) and np.array_equal(g[2], w[2])


def test_arguments(tmp_path):
    det = _detector("fp16x2", "dla_34")
    with pytest.raises(FileNotFoundError):
        det.run_video(str(tmp_path / "missing.mp4"))
    with pytest.raises(ValueError, match="encode_png"):
        det.run_video([], encode_png=True)
    with pytest.raises(ValueError, match="max_batch"):
        det.run_video([], max_batch=0)
    assert list(det.run_video([])) == []
    # a caller that stops early leaves no reader thread behind
    frames = [rc.image(120, 160, k) for k in range(6)]
    gen = det.run_video(iter(frames), max_batch=2)
    next(gen)
    gen.close()
    assert not reader_threads()


def test_device_polygons_equal_model():
    from centerpose_b200 import _lib
    from tests import ellipse_model as em
    cx, cy, L = em.domain()
    n = len(L)
    verts = torch.empty((n, em.MAX_POINTS, 2), dtype=torch.int32, device="cuda")
    counts = torch.empty(n, dtype=torch.int32, device="cuda")
    for angle in range(-180, 181):
        params = torch.from_numpy(np.stack([cx, cy, L, np.full(n, angle)], 1).astype(np.int32)).cuda()
        _lib.launch("ellipse_poly_batch", torch.device("cuda"), params, n, verts, counts)
        pts, want = em.ellipse_polys(cx, cy, L, angle)
        got_counts = counts.cpu().numpy()
        assert np.array_equal(got_counts, want), angle
        v = verts.cpu().numpy()
        got = v[np.arange(em.MAX_POINTS)[None] < got_counts[:, None]]
        assert np.array_equal(got, pts), angle


def _border_rows(h, w):
    """Persons whose label boxes the left, right and bottom borders cut (edge_rows cuts the top)."""
    r = rc.rows(h, w, 6, 77)
    r[:, 4] = 0.62
    r[0, :4] = (-12, h // 2, 20, h // 2 + 30)                # text starts left of column 0
    r[1, :4] = (w - 15, h // 2, w + 20, h // 2 + 30)         # text runs past the right border
    r[2, :4] = (w // 3, h + 6, w // 2, h + 40)               # label box below the image, text partly in
    r[3, :4] = (w // 3, h + 1, w // 2, h + 40)
    r[4, :4] = (w - 4, 3, w + 40, 20)                        # cut right and top
    r[5, 4] = 0.3                                             # at the threshold: not drawn
    return r


@pytest.mark.parametrize("theme", ["white", "black"])
@pytest.mark.parametrize("h,w", [(120, 160), (359, 641)])
def test_device_plan_draws_as_render_poses(h, w, theme):
    from centerpose_b200 import render
    det = _detector("fp16x2", "dla_34")
    det.cfg.DEBUG_THEME = theme
    det.cfg.TEST.VIS_THRESH = 0.3
    try:
        B, N = 5, 48
        rows = np.zeros((B, N, 56), np.float32)
        for b in range(B):
            r = np.concatenate([rc.rows(h, w, 30, 300 + b, off=0.4), rc.edge_rows(h, w), _border_rows(h, w)])
            rows[b, :len(r)] = r
        rows[1, :, 4] = 0.0                                    # an image that draws nothing
        images = [rc.image(h, w, 400 + b) for b in range(B)]
        want = det.render_poses(images, list(rows))
        for first_share in (1 << 14, 16):                      # 16 vertices: the plan outgrows its share and re-runs
            plan = render.DevicePlan(0.3, theme, torch.device("cuda"))
            plan.verts_per_image, plan.rows_per_image = first_share, first_share * 8
            pixels = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).cuda()
            plan.draw(plan.plan(torch.from_numpy(rows).cuda(), h, w), pixels)
            got = pixels.cpu().numpy().reshape(B, h, w, 3)
            for b in range(B):
                assert np.array_equal(got[b], want[b]), (first_share, b)
    finally:
        det.cfg.DEBUG_THEME = "white"
        det.cfg.TEST.VIS_THRESH = 0.05


def test_device_plan_errors():
    from centerpose_b200 import render
    plan = render.DevicePlan(0.3, "white", torch.device("cuda"))
    rows = np.zeros((1, 2, 56), np.float32)
    rows[0, 0, 4] = np.inf
    with pytest.raises(ValueError, match="finite"):
        plan.draw(plan.plan(torch.from_numpy(rows).cuda(), 50, 60), torch.zeros(50 * 60 * 3, dtype=torch.uint8).cuda())
    det = _detector("fp16x2", "dla_34")
    det.cfg.TEST.VIS_THRESH = -1.0
    try:
        with pytest.raises(ValueError, match="VIS_THRESH"):
            det.run_video([], return_images=True)
    finally:
        det.cfg.TEST.VIS_THRESH = 0.05
