"""Annotation sets for the validation-target tests: ``constructed()`` and the seeded ``random_case(seed)``.

Each case is a single-category COCO keypoint dict with one image per entry (``images`` carry ``height`` and
``width``).  The constructed images reach: crowd and zero-keypoint objects, an image whose objects are all crowds, more
than 32 objects, boxes across the image edge, boxes that clip to h = 0 or w = 0, joints outside the output and joints
with v = 0 but coordinates, radius-0 and largest-radius boxes, overlapping stamps, landscape, portrait, square and odd
sizes (an odd width puts c on a half pixel), and trans_output matrices with non-zero off-diagonals.
"""
from __future__ import annotations

import numpy as np

J = 17


def _ann(ann_id, image_id, bbox, kps, crowd=0):
    kps = np.asarray(kps, np.float64).reshape(J, 3)
    return {"id": int(ann_id), "image_id": int(image_id), "category_id": 1, "iscrowd": int(crowd),
            "bbox": [float(v) for v in bbox], "area": float(bbox[2] * bbox[3]),
            "keypoints": [float(v) if v != int(v) else int(v) for v in kps.reshape(-1)],
            "num_keypoints": int(np.count_nonzero(kps[:, 2] > 0))}


def _person(rng, x, y, w, h, vis="full"):
    kx = x + rng.random(J) * w
    ky = y + rng.random(J) * h
    if vis == "full":
        v = np.full(J, 2.0)
    elif vis == "none":
        v = np.zeros(J)
    else:
        v = rng.choice([0.0, 1.0, 2.0], J)
    if vis == "none":
        kx[:] = ky[:] = 0.0
    return np.stack([np.round(kx, 2), np.round(ky, 2), v], 1)


def _dataset(images, anns):
    return {"categories": [{"id": 1, "name": "person"}],
            "images": [{"id": i, "height": h, "width": w, "file_name": "%d.png" % i} for i, h, w in images],
            "annotations": anns}


def constructed():
    """The constructed annotation sets as one dataset."""
    rng = np.random.default_rng(7)
    images, anns = [], []
    aid = [1]

    def add(image_id, bbox, kps, crowd=0):
        anns.append(_ann(aid[0], image_id, bbox, kps, crowd))
        aid[0] += 1

    # 1: landscape, crowds between ordinary objects, a zero-keypoint object, overlapping people
    images.append((1, 480, 640))
    add(1, [100, 80, 120, 300], _person(rng, 100, 80, 120, 300))
    add(1, [0, 0, 640, 480], _person(rng, 0, 0, 640, 480, "none"), crowd=1)
    add(1, [150, 90, 110, 280], _person(rng, 150, 90, 110, 280, "partial"))
    add(1, [400, 200, 60, 150], _person(rng, 400, 200, 60, 150, "none"))
    add(1, [420, 210, 55, 140], _person(rng, 420, 210, 55, 140))
    # 2: only crowds: nothing kept
    images.append((2, 300, 400))
    add(2, [10, 10, 200, 200], _person(rng, 10, 10, 200, 200), crowd=1)
    add(2, [50, 50, 100, 100], _person(rng, 50, 50, 100, 100, "none"), crowd=1)
    # 3: portrait, more than 32 objects (a crowd among them), small boxes: radius 0 and 1
    images.append((3, 641, 427))
    for n in range(40):
        x, y = 10 + (n % 8) * 50, 10 + (n // 8) * 120
        size = [2, 3, 5, 8, 13][n % 5]
        add(3, [x, y, size, size * 2], _person(rng, x, y, size, size * 2, "partial"), crowd=int(n == 5))
    # 4: square, a largest-radius box, boxes across every edge, a box left of the image (w clips to 0) and one below
    #    it (h clips to 0), joints outside the output, joints with v = 0 but coordinates
    images.append((4, 512, 512))
    add(4, [0, 0, 512, 512], _person(rng, 0, 0, 512, 512))
    add(4, [-40, 100, 120, 200], _person(rng, -60, 100, 160, 200))
    add(4, [450, -30, 100, 120], _person(rng, 430, -60, 140, 160))
    add(4, [-100, 50, 60, 100], _person(rng, -100, 50, 60, 100))
    add(4, [100, 600, 80, 90], _person(rng, 100, 600, 80, 90))
    hidden = _person(rng, 200, 200, 100, 200, "none")
    hidden[:, 0:2] = _person(rng, 200, 200, 100, 200)[:, 0:2]
    add(4, [200, 200, 100, 200], hidden)
    mixed = _person(rng, 300, 300, 150, 150, "partial")
    mixed[mixed[:, 2] == 0, 0:2] = [[333.5, 350.25]]
    add(4, [300, 300, 150, 150], mixed)
    # 5: odd sizes (c on half pixels), fractional boxes
    images.append((5, 333, 517))
    add(5, [12.37, 40.91, 200.5, 250.75], _person(rng, 12.37, 40.91, 200.5, 250.75))
    add(5, [300.01, 10.99, 0.49, 100.3], _person(rng, 300.01, 10.99, 0.49, 100.3, "partial"))
    add(5, [510.5, 320.5, 30.2, 40.1], _person(rng, 505, 315, 30, 30, "partial"))
    # 6..: sizes whose trans_output has non-zero off-diagonal entries
    for image_id, (h, w) in enumerate(OFF_DIAGONAL_SHAPES, start=6):
        images.append((image_id, h, w))
        for n in range(4):
            x, y = rng.uniform(0, w - 40), rng.uniform(0, h - 40)
            bw, bh = rng.uniform(5, w - x), rng.uniform(5, h - y)
            add(image_id, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)],
                _person(rng, x, y, bw, bh, "partial"))
    return _dataset(images, anns)


# image sizes (h, w) for which get_affine_transform(c, s, 0, [128, 128]) has non-zero off-diagonal entries
OFF_DIAGONAL_SHAPES = [(100, 347), (100, 503), (100, 685)]


def random_case(seed, n_images=4):
    """A seeded dataset of ``n_images`` images of random size with 0..40 random annotations each: crowds, hidden
    and zero-keypoint objects, boxes partly or wholly outside the image, joints anywhere around it."""
    rng = np.random.default_rng(1000 + seed)
    images, anns = [], []
    aid = 1
    for i in range(n_images):
        h, w = int(rng.integers(16, 800)), int(rng.integers(16, 800))
        images.append((i + 1, h, w))
        for _ in range(int(rng.integers(0, 41))):
            bw, bh = rng.uniform(0.1, 1.2) * w, rng.uniform(0.1, 1.2) * h
            if rng.random() < 0.3:
                bw, bh = rng.uniform(0, 12), rng.uniform(0, 12)
            x, y = rng.uniform(-0.3 * w, w), rng.uniform(-0.3 * h, h)
            kps = _person(rng, x - 0.1 * bw, y - 0.1 * bh, 1.2 * bw, 1.2 * bh,
                          rng.choice(["full", "partial", "partial", "none"]))
            if rng.random() < 0.2:
                kps[:, 0:2] = np.round(rng.uniform(-50, max(h, w) + 50, (J, 2)), 2)
            anns.append(_ann(aid, i + 1, [round(x, 2), round(y, 2), round(bw, 2), round(bh, 2)], kps,
                             crowd=int(rng.random() < 0.1)))
            aid += 1
    return _dataset(images, anns)


def shapes_of(ds):
    """``{image_id: (h, w)}`` of a case."""
    return {im["id"]: (im["height"], im["width"]) for im in ds["images"]}
