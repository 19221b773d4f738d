"""GPU tests of the PNG encoder (cpb200_png_encode_batch): png.encode and run_images(..., encode_png=True) against
cv2.imencode('.png', ...), byte for byte."""
import cv2
import numpy as np
import pytest
import torch

from centerpose_b200 import heatmaps, png, render
from tests import png_encode_cases as pc
from tests import render_cases as rc

pytestmark = pytest.mark.gpu

_DET = {}


def cv2_png(img):
    return cv2.imencode(".png", np.ascontiguousarray(img))[1].tobytes()


def coco_drawn(n):
    """COCO-sized images with poses drawn by render_poses."""
    shapes = [(480, 640), (427, 640), (640, 480), (375, 500)]
    imgs = [rc.image(*shapes[k % 4], 100 + k) for k in range(n)]
    rows = [rc.rows(*shapes[k % 4], 12, 200 + k) for k in range(n)]
    shapes = [im.shape[:2] for im in imgs]
    pixels, offsets = render.launch(render.build(shapes, rows, 0.3, "white"), images=imgs)
    return render.download(pixels, offsets, shapes)


def coco_views(n):
    """Both heat-map views of n 512 x 512 network inputs."""
    rng = np.random.default_rng(7)
    x = [torch.from_numpy(rng.normal(0, 1, (3, 512, 512)).astype(np.float32)).cuda() for _ in range(n)]
    hm = [torch.from_numpy(rng.random((1, 128, 128)).astype(np.float32) ** 4).cuda() for _ in range(n)]
    hp = [torch.from_numpy(rng.random((17, 128, 128)).astype(np.float32) ** 6).cuda() for _ in range(n)]
    views = heatmaps.views(x, hm, hp, 4, "white", np.array([0.408, 0.447, 0.470]), np.array([0.289, 0.274, 0.278]))
    return [v[k] for v in views for k in heatmaps.VIEWS]


def test_encode_matrix_one_launch():
    imgs = [img for _, img in pc.cases()] + coco_drawn(4) + coco_views(2)
    got = png.encode(imgs)
    bad = [i for i, (g, img) in enumerate(zip(got, imgs)) if g != cv2_png(img)]
    assert not bad, "differ from cv2.imencode: %s" % [pc.cases()[i][0] if i < len(pc.cases()) else i for i in bad]


def test_packed_output_leaves_guard_bytes():
    imgs = [img for _, img in pc.cases()[:20]]
    srcs = [torch.from_numpy(img).cuda() for img in imgs]
    table, counts, ws, out_bytes = png.encode_layout([t.data_ptr() for t in srcs], [i.shape[:2] for i in imgs],
                                                     [3 * i.shape[1] for i in imgs])
    assert out_bytes >= sum(len(cv2_png(i)) for i in imgs)
    out = torch.full((out_bytes + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(len(imgs), dtype=torch.int64, device="cuda")
    png.encode_launch(table, counts, ws, out, sizes)
    files = png.download_files(out, sizes)
    assert files == [cv2_png(i) for i in imgs]
    total = int(sizes.sum())
    assert bool((out[total:] == 0xA5).all())


def test_alone_and_in_batch_and_tensor_inputs_agree():
    cases = pc.cases()
    img = cases[-1][1]
    alone = png.encode([img])[0]
    batch = png.encode([cases[3][1], img, cases[10][1]])[1]
    cuda = png.encode([torch.from_numpy(img).cuda()])[0]
    # a CUDA view with a row pitch wider than the row
    wide = torch.zeros((img.shape[0], img.shape[1] + 5, 3), dtype=torch.uint8, device="cuda")
    wide[:, :img.shape[1]] = torch.from_numpy(img).cuda()
    pitched = png.encode([wide[:, :img.shape[1]]])[0]
    assert alone == batch == cuda == pitched == cv2_png(img)


@pytest.mark.parametrize("bad", ["float", "gray", "four", "empty", "list", "cpu_tensor"])
def test_encode_rejects(bad):
    img = {"float": np.zeros((4, 4, 3), np.float32), "gray": np.zeros((4, 4), np.uint8),
           "four": np.zeros((4, 4, 4), np.uint8), "empty": np.zeros((0, 4, 3), np.uint8),
           "list": [[1, 2, 3]], "cpu_tensor": torch.zeros((4, 4, 3), dtype=torch.uint8)}[bad]
    with pytest.raises(ValueError):
        png.encode([np.zeros((2, 2, 3), np.uint8), img])


def _detector():
    from centerpose_b200.config import default_cfg
    from centerpose_b200.detector import detector_factory
    from oracle.init_recipe import conditioned_state_dict
    if "det" not in _DET:
        cfg = default_cfg("dla_34")
        det = detector_factory[cfg.TEST.TASK](cfg)
        det.model.load_state_dict(conditioned_state_dict(det.model.state_dict(), 317))
        _DET["det"] = det
    det = _DET["det"]
    det.cfg.TEST.VIS_THRESH = 0.05
    return det


def test_run_images_encode_png(tmp_path):
    det = _detector()
    arrays = [rc.image(480, 640, 11), rc.image(360, 500, 12)]
    paths = []
    for k, (ext, img) in enumerate(zip((".jpg", ".png"), (rc.image(427, 640, 13), rc.image(300, 420, 14)))):
        p = str(tmp_path / ("im%d%s" % (k, ext)))
        cv2.imwrite(p, img)
        paths.append(p)
    for images in (arrays, arrays + paths):
        rows, drawn, views = det.run_images(images, return_images=True, return_heatmaps=True)
        rows2, drawn_png, views_png = det.run_images(images, return_images=True, return_heatmaps=True,
                                                     encode_png=True)
        assert all(np.array_equal(a, b) for a, b in zip(rows, rows2))
        assert [type(d) for d in drawn_png] == [bytes] * len(images)
        assert drawn_png == [cv2_png(d) for d in drawn]
        assert views_png == [{k: cv2_png(v[k]) for k in heatmaps.VIEWS} for v in views]
    rows, drawn_png = det.run_images(arrays, return_images=True, encode_png=True)
    assert drawn_png == [cv2_png(d) for d in det.run_images(arrays, return_images=True)[1]]
    rows, views_png = det.run_images(arrays, return_heatmaps=True, encode_png=True)
    assert views_png == [{k: cv2_png(v[k]) for k in heatmaps.VIEWS}
                         for v in det.run_images(arrays, return_heatmaps=True)[1]]


def test_run_images_encode_png_needs_images():
    with pytest.raises(ValueError):
        _detector().run_images([rc.image(64, 64, 1)], encode_png=True)
