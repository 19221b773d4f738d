"""The PNG encoder without a GPU: tests/png_encode_model.py (the device stages in numpy / Python) against
cv2.imencode('.png', ...) and zlib byte for byte on a matrix that reaches every branch of the format, the facts the
device relies on, and the host layout of a launch."""
from __future__ import annotations

import zlib

import cv2
import numpy as np
import pytest

from centerpose_b200 import png
from oracle import debugger_ref, heatmaps_ref
from tests import png_encode_cases as pc
from tests import png_encode_model as M
from tests import render_cases as rc

CASES = pc.cases()


def coco_images():
    """COCO-sized drawn poses (the reference Debugger's drawing) and heat-map views of a 512 x 512 input."""
    out = []
    for k, (h, w) in enumerate(((480, 640), (427, 640))):
        out.append(("drawn_%dx%d" % (h, w), debugger_ref.show_results(rc.image(h, w, 30 + k),
                                                                      rc.rows(h, w, 12, 40 + k).tolist(), 0.3, "white")))
    rng = np.random.default_rng(3)
    x = rng.normal(0, 1, (3, 512, 512)).astype(np.float32)
    hm = (rng.random((1, 128, 128)) ** 4).astype(np.float32)
    hp = (rng.random((17, 128, 128)) ** 6).astype(np.float32)
    views = heatmaps_ref.heatmap_views(x, hm, hp, 4, "white", np.array([0.408, 0.447, 0.470], np.float32),
                                       np.array([0.289, 0.274, 0.278], np.float32))
    return out + [("view_" + k, v) for k, v in views.items()]


def cv2_png(img):
    return cv2.imencode(".png", img)[1].tobytes()


def trace(img):
    f = M.filtered(img)
    t = []
    M.deflate(f, t)
    return f, t


@pytest.mark.parametrize("name,img", CASES + coco_images(), ids=lambda v: v if isinstance(v, str) else "")
def test_model_equals_cv2(name, img):
    assert M.png(img) == cv2_png(img)


@pytest.mark.parametrize("name,img", CASES, ids=lambda v: v if isinstance(v, str) else "")
def test_model_equals_zlib(name, img):
    """zlib.compressobj at level 1, Z_RLE, memLevel 8 and libpng's window over the whole scanline buffer writes the
    same stream: libpng's row-by-row feeding changes nothing, and only the header differs (optimize_cmf)."""
    f = M.filtered(img)
    co = zlib.compressobj(1, zlib.DEFLATED, M.window_bits(f.size), 8, zlib.Z_RLE)
    z = co.compress(f.tobytes()) + co.flush()
    assert z[2:] == M.zstream(img)[2:]


def test_matrix_reaches_every_branch():
    header, kinds, last_sizes, zmod, lengths = set(), set(), set(), set(), set()
    ties = overflow = run_over_block = 0
    widths = set()
    for name, img in CASES:
        f, t = trace(img)
        widths.add(img.shape[1])
        lengths.add(f.size)
        header.add(M.zlib_header(f.size))
        kinds |= {k for k, *_ in t}
        last_sizes.add(t[-1][1])
        zmod.add(len(M.zstream(img)) % M.IDAT_BYTES)
        ties += sum((c.opt_len + 10) >> 3 == (c.static_len + 10) >> 3 for *_, c in t)
        overflow += sum(c.overflowed for *_, c in t)
        sym = M.symbols(f)
        ends = np.cumsum(M.symbol_bytes(sym))
        for b in range(1, len(t)):
            k = b * M.BLOCK_SYMBOLS
            if k < sym.size and f[ends[k - 1] - 1] == f[ends[k - 1]]:
                run_over_block += 1
    assert 1 in widths
    assert {bytes.fromhex(h) for h in ("7801", "6805", "5809", "1819", "081d")} <= header
    assert {16384, 16385} <= lengths
    assert kinds == {"stored", "static", "dynamic"}
    assert {0, 1} <= last_sizes                  # an empty final block, a final block of one symbol
    assert 0 in zmod                             # a zlib stream of exactly 3 IDAT chunks
    assert ties and overflow and run_over_block


def test_runs_decompose_in_closed_form():
    for L in range(1, 800):
        f = np.r_[np.uint8(7), np.zeros(L, np.uint8), np.uint8(9)]
        sym = M.symbols(f)[1:-1]
        q, r = divmod(L - 1, 258)
        want = [0] + [256 + 255] * q + ([256 + r - 3] if r >= 3 else [0] * r)
        assert sym.tolist() == want


def test_stored_block_start_stays_in_the_window():
    """zlib may store a block only while its start is in the window.  Below 16 KiB of scanlines the window holds them
    all; above, a block leaves it only when it covers more than 32 506 bytes, and then storing never wins."""
    for name, img in CASES + coco_images():
        f, t = trace(img)
        if f.size <= 16384:
            assert f.size + 262 <= 1 << M.window_bits(f.size)
        for kind, nsym, stored_len, c in t:
            if stored_len > 32506:
                assert stored_len + 4 > (c.static_len + 10) >> 3, name


def test_layout_bounds_and_table():
    shapes = [img.shape[:2] for _, img in CASES]
    pitches = [3 * w + 8 * k for k, (h, w) in enumerate(shapes)]
    table, (tiles, blocks, chunks), ws, out = png.encode_layout([0x1000 * (k + 1) for k in range(len(shapes))],
                                                                shapes, pitches)
    assert out == sum(png.encode_bound(h, w) for h, w in shapes)
    for (name, img), e in zip(CASES, table):
        f = M.filtered(img)
        n = f.size
        assert png.encode_bound(*img.shape[:2]) >= len(cv2_png(img))
        assert e["z_bytes"] >= len(M.zstream(img)) + 8 and e["z_bytes"] % 16 == 0
        assert (e["h"], e["w"]) == img.shape[:2] and e["pitch"] >= 3 * e["w"]
        assert e["z_offset"] % 16 == 0 and e["sym_offset"] % 2 == 0
        assert e["tile_offset"] % 8 == 0 and e["block_offset"] % 8 == 0 and e["state_offset"] % 8 == 0
        spans = sorted([(e["filt_offset"], n), (e["sym_offset"], 2 * n), (e["tile_offset"], -(-n // 4096) * 32),
                        (e["block_offset"], (n // 16383 + 1) * 1088), (e["state_offset"], 64),
                        (e["z_offset"], e["z_bytes"])])
        assert all(a + s <= b for (a, s), (b, _) in zip(spans, spans[1:]))
        assert spans[-1][0] + spans[-1][1] <= ws
        assert M.symbols(f).size // M.BLOCK_SYMBOLS + 1 <= n // 16383 + 1
    for field, total in (("tile0", tiles), ("block0", blocks), ("chunk0", chunks)):
        firsts = table[field].tolist() + [total]
        assert firsts[0] == 0 and all(a < b for a, b in zip(firsts, firsts[1:]))
    assert np.diff(table["chunk0"]).tolist() + [chunks - table["chunk0"][-1]] == \
        [-(-int(z) // 8192) for z in table["z_bytes"]]


@pytest.mark.parametrize("bad", [np.zeros((4, 4, 3), np.float32), np.zeros((4, 4), np.uint8),
                                 np.zeros((4, 4, 4), np.uint8), np.zeros((0, 4, 3), np.uint8),
                                 np.zeros((4, 0, 3), np.uint8), [[1, 2, 3]]])
def test_encode_rejects_before_any_launch(bad):
    with pytest.raises(ValueError):
        png.encode([np.zeros((2, 2, 3), np.uint8), bad])
