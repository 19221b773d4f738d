"""The pose drawing without a GPU: the oracle against the reference's Debugger (golden), cv2's rasterisation rules
(``tests/render_model.py``) against cv2, the text tables, the addWeighted model, and the launch tables of
``centerpose_b200.render.build`` replayed in numpy against the oracle."""
from __future__ import annotations

import math
import os

import cv2
import numpy as np
import pytest

from centerpose_b200 import render
from oracle import debugger_ref
from tests import render_cases as rc
from tests import render_model as rm

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "render_poses.npz")


def golden_cases():
    g = np.load(GOLDEN)
    n = len([k for k in g.files if k.startswith("out_")])
    return [(g["image_%d" % k], g["rows_%d" % k], str(g["theme_%d" % k]), g["out_%d" % k]) for k in range(n)]


def replay(image, ops, i=0):
    """``render_poses_kernel``'s steps on image i of ``ops`` in numpy, with tests/render_model.py's pixel sets."""
    img = image.copy()
    h, w = img.shape[:2]
    im = ops.images[i]
    for p in ops.persons[im["person_begin"]:im["person_begin"] + im["person_count"]]:
        c = p["color"][:3]
        img[rm.rect_mask(w, h, *[int(v) for v in p["box"]])] = c
        lx0, ly0, lx1, ly1 = [int(v) for v in p["label"]]
        m = np.zeros((h, w), bool)
        rm._fill(m, min(lx0, lx1), min(ly0, ly1), max(lx0, lx1), max(ly0, ly1))
        img[m] = c
        luts = ops.luts.reshape(-1)
        for t in ops.text_px[p["text_begin"]:p["text_begin"] + p["text_count"]]:
            y, x = p["text_y"] + t["dy"], p["text_x"] + t["dx"]
            img[y, x] = luts[t["lut"] + img[y, x].astype(np.int64)]
        for j in range(17):
            if p["joints"] >> j & 1:
                img[rm.circle2_mask(w, h, int(p["joint_x"][j]), int(p["joint_y"][j]))] = 255
        n = p["limb_count"]
        first = np.full((h, w), 255, np.int64)
        for r, L in enumerate(ops.limbs[p["limb_begin"]:p["limb_begin"] + n]):
            v = ops.verts[2 * L["vert_begin"]:2 * (L["vert_begin"] + L["vert_count"])].reshape(-1, 2)
            m = rm.convex_mask(w, h, [tuple(q) for q in v]) & (first == 255)
            first[m] = r
        fold = np.arange(256)[None].repeat(19, 0)
        for k in range(1, 19):
            fold[k] = blend_model(fold[k - 1], 255)
        hit = first != 255
        img[hit] = fold[n - first[hit][:, None], img[hit]]
    return img


def blend_model(v, c):
    s = np.float32(np.asarray(v, np.float32) * np.float32(0.8)) + np.float32(np.asarray(c, np.float32) * np.float32(0.2))
    return np.clip(np.rint(s.astype(np.float32)), 0, 255).astype(np.uint8)


def test_oracle_equals_golden():
    cases = golden_cases()
    assert {t for _, _, t, _ in cases} == {"white", "black"}
    for img, rows, theme, out in cases:
        assert np.array_equal(debugger_ref.show_results(img, rows.tolist(), 0.3, theme), out)


def test_golden_covers_the_cases():
    cases = golden_cases()
    rows = np.concatenate([r for _, r, _, _ in cases])
    drawn = rows[rows[:, 4].astype(np.float64) > 0.3]
    assert {render.label_text(s) for s in drawn[:, 4]} == {"p%.1f" % (k / 10) for k in range(3, 11)}
    assert (rows[:, 4] == np.float32(0.3)).any()                       # just above VIS_THRESH as a double
    assert (drawn[:, 39:] <= 0).any() and (drawn[:, 39:] > 0).any()
    assert (drawn[:, 1] < 14).any()                                     # label boxes cut by the top row
    assert any(((r[:, 0] < 0) | (r[:, 2] >= img.shape[1])).any() for img, r, _, _ in cases)


def test_table_replay_equals_golden():
    for img, rows, theme, out in golden_cases():
        ops = render.build([img.shape[:2]], [rows], 0.3, theme)
        assert np.array_equal(replay(img, ops), out)


@pytest.mark.parametrize("seed", range(2))
def test_table_replay_equals_oracle(seed):
    h, w = [(97, 131), (33, 200)][seed]
    img = rc.image(h, w, seed)
    rows = np.concatenate([rc.rows(h, w, 10, seed, spread=0.7, off=0.4), rc.edge_rows(h, w)])
    rows[:, 4] = np.where(rows[:, 4] > 0.3, rows[:, 4], 0.9)
    for theme in ("white", "black"):
        ops = render.build([img.shape[:2]], [rows], 0.3, theme)
        assert np.array_equal(replay(img, ops), debugger_ref.show_results(img, rows.tolist(), 0.3, theme))


def test_limb_geometry_matches_reference_arithmetic():
    rng = np.random.default_rng(5)
    for _ in range(3000):
        pts = rng.integers(-3000, 3000, (17, 2)).astype(np.int32)
        if rng.random() < 0.2:
            pts[1] = pts[0]
        a, b = render.EDGES[rng.integers(len(render.EDGES))]
        X = [pts[a, 1], pts[b, 1]]
        Y = [pts[a, 0], pts[b, 0]]
        length = ((X[0] - X[1]) ** 2 + (Y[0] - Y[1]) ** 2) ** 0.5
        angle = math.degrees(math.atan2(X[0] - X[1], Y[0] - Y[1]))
        want = cv2.ellipse2Poly((int(np.mean(Y)), int(np.mean(X))), (int(length / 2), 2), int(angle), 0, 360, 1)
        assert np.array_equal(render.limb_polygon(pts, a, b), want)


def test_label_box_and_int32_truncation():
    row = np.zeros(56, np.float32)
    row[:5] = (10.9, -3.7, 40.2, 30.999, 0.55)
    ops = render.build([(20, 30)], [row[None]], 0.3)
    p = ops.persons[0]
    (tw, th), _ = cv2.getTextSize("p0.6", cv2.FONT_HERSHEY_SIMPLEX, 0.5, 2)
    assert list(p["box"]) == [10, -3, 40, 30]
    assert list(p["label"]) == [10, -3 - th - 2, 10 + tw, -5]
    assert p["text_count"] == 0                                        # the whole label is above row 0
    assert render.label_text(np.float32(0.55)) == "p0.6" and render.label_text(0.25) == "p0.2"


def test_vis_thresh_is_strict():
    rows = np.zeros((3, 56), np.float32)
    rows[:, 4] = (0.3, np.nextafter(np.float32(0.3), np.float32(0)), 0.2)    # float32 0.3 is above 0.3 as a double
    ops = render.build([(20, 30)], [rows], 0.3)
    assert len(ops.persons) == 1 and list(ops.persons[0]["box"]) == [0, 0, 0, 0]


def test_text_tables_on_random_backgrounds():
    rng = np.random.default_rng(9)
    for k in range(60):
        txt = "p%.1f" % (k % 11 / 10)
        h, w = [int(v) for v in rng.integers(1, 40, 2)]
        ox, oy = [int(v) for v in rng.integers(-40, 60, 2)]
        bg = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        want = bg.copy()
        cv2.putText(want, txt, (ox, oy), cv2.FONT_HERSHEY_SIMPLEX, 0.5, (0, 0, 0), 1, cv2.LINE_AA)
        x0, x1, y0, y1 = render._text_extent(txt)
        ax, bx, ay, by = max(-ox, x0), min(w - 1 - ox, x1), max(-oy, y0), min(h - 1 - oy, y1)
        got = bg.copy()
        if ax <= bx and ay <= by:
            dx, dy, luts = render.text_table(txt, ax, bx, ay, by)
            for a, b, lut in zip(dx, dy, luts):
                got[oy + b, ox + a] = lut[got[oy + b, ox + a]]
        assert np.array_equal(got, want), (txt, h, w, ox, oy)


def test_add_weighted_model_all_pairs():
    v, c = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    want = cv2.addWeighted(v, 0.8, c, 0.2, 0)
    assert np.array_equal(blend_model(v, c), want)
    assert np.array_equal(blend_model(v, v), v)                         # a blend with an unchanged canvas is a no-op


def test_line_and_convex_fill_model():
    rng = np.random.default_rng(2)
    for t in range(1500):
        h, w = [int(v) for v in rng.integers(1, 60, 2)]
        s = [10, 80, 1000, 10 ** 6][t % 4]
        x1, y1, x2, y2 = [int(v) for v in rng.integers(-s, s + 60, 4)]
        img = np.zeros((h, w), np.uint8)
        cv2.line(img, (x1, y1), (x2, y2), 255, 1, cv2.LINE_8)
        m = np.zeros((h, w), bool)
        for x, y in rm.line_pixels(w, h, x1, y1, x2, y2):
            m[y, x] = True
        assert np.array_equal(img > 0, m), ("line", h, w, x1, y1, x2, y2)
        s = [10, 80, 300, 3000][t % 4]
        cx, cy = [int(v) for v in rng.integers(-s, 60 + s, 2)]
        length = int(rng.integers(0, [5, 40, 200, 3000][(t // 4) % 4]))
        pts = cv2.ellipse2Poly((cx, cy), (length, 2), int(rng.integers(-180, 181)), 0, 360, 1)
        img = np.zeros((h, w), np.uint8)
        cv2.fillConvexPoly(img, pts, 255)
        assert np.array_equal(img > 0, rm.convex_mask(w, h, [tuple(p) for p in pts])), ("ellipse", h, w, cx, cy)
        k = int(rng.integers(1, 9))
        P = rng.integers(-[5, 50, 500][t % 3], [5, 50, 500][t % 3] + 60, (k, 2)).astype(np.int32)
        hull = cv2.convexHull(P).reshape(-1, 2) if k >= 3 else P
        img = np.zeros((h, w), np.uint8)
        cv2.fillConvexPoly(img, hull, 255)
        assert np.array_equal(img > 0, rm.convex_mask(w, h, [tuple(p) for p in hull])), ("hull", h, w, hull.tolist())


def test_rectangle_and_disc_model():
    rng = np.random.default_rng(1)
    for t in range(2500):
        h, w = [int(v) for v in rng.integers(1, 40, 2)]
        s = [3, 40, 100, 3000, 100000][t % 5]       # cv2 walks every row above the image, so far-off boxes are slow
        x1, y1, x2, y2 = [int(v) for v in rng.integers(-s, s + 40, 4)]
        if t % 7 == 0:
            x2 = x1
        if t % 11 == 0:
            y2 = y1
        img = np.zeros((h, w), np.uint8)
        cv2.rectangle(img, (x1, y1), (x2, y2), 255, 2)
        assert np.array_equal(img > 0, rm.rect_mask(w, h, x1, y1, x2, y2)), ("rect", h, w, x1, y1, x2, y2)
        img = np.zeros((h, w), np.uint8)
        cv2.rectangle(img, (x1, y1), (x2, y2), 255, -1)
        m = np.zeros((h, w), bool)
        rm._fill(m, min(x1, x2), min(y1, y2), max(x1, x2), max(y1, y2))
        assert np.array_equal(img > 0, m), ("filled rect", h, w, x1, y1, x2, y2)
        x, y = [int(v) for v in rng.integers(-[5, 100, 2 ** 30][t % 3], [5, 100, 2 ** 30][t % 3] + 12, 2)]
        img = np.zeros((h, w), np.uint8)
        cv2.circle(img, (x, y), 2, 255, -1)
        assert np.array_equal(img > 0, rm.circle2_mask(w, h, x, y)), ("disc", h, w, x, y)
