"""The heat-map views without a GPU: the oracle against the reference's Debugger (golden), the launch table of
``centerpose_b200.heatmaps`` replayed in numpy with the kernels' integer resize and the numpy cast they copy, and the
argument checks that run before any launch."""
from __future__ import annotations

import os

import numpy as np
import pytest
import torch

from centerpose_b200 import heatmaps
from oracle import heatmaps_ref
from tests.test_resize_cpu import resize_linear

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "heatmap_views.npz")
THEMES = ("white", "black")


def golden_cases():
    """``(x, hm, hm_hp, dr, {theme: {view: image}})`` per case, and the golden's mean and std."""
    g = np.load(GOLDEN)
    n = len([k for k in g.files if k.startswith("x_")])
    cases = [(g["x_%d" % k], g["hm_%d" % k], g["hp_%d" % k], int(g["dr_%d" % k]),
              {t: {v: g["%s_%s_%d" % (t, v, k)] for v in heatmaps.VIEWS} for t in THEMES}) for k in range(n)]
    return cases, g["mean"], g["std"]


def numpy_u8(v):
    """The cast ``numpy_u8`` in csrc/heatmaps.cu: truncate to int32 and keep the low 8 bits; NaN and |v| >= 2^31
    give 0."""
    v = np.asarray(v, np.float32)
    ok = (v > -2.0 ** 31) & (v < 2.0 ** 31)
    return np.where(ok, np.trunc(np.where(ok, v, 0)).astype(np.int64) & 255, 0).astype(np.uint8)


def replay(table, bases, out_bytes, ws_bytes, theme, mean, std):
    """What the three kernels do with ``table``, in numpy: ``bases`` are the tensors the table's addresses point
    into.  Returns the output bytes; asserts every read and every workspace region lies where it should."""
    def read(ptr, n):
        for t in bases:
            start = t.data_ptr()
            if start <= ptr and ptr + 4 * n <= start + 4 * t.numel():
                assert (ptr - start) % 4 == 0
                return t.numpy().reshape(-1)[(ptr - start) // 4:(ptr - start) // 4 + n]
        raise AssertionError("table address %#x is in no source tensor" % ptr)

    colors = heatmaps.colors(theme)
    out = np.zeros(out_bytes, np.uint8)
    ws_used = np.zeros(ws_bytes, bool)
    out_used = np.zeros(out_bytes, bool)
    for e in table:
        H, W, h, w, C, dr = (int(e[k]) for k in ("H", "W", "h", "w", "C", "dr"))
        x = read(int(e["input"]), 3 * H * W).reshape(3, H, W)
        ws = slice(int(e["ws_offset"]), int(e["ws_offset"]) + 2 * (h * w + H * W) * 3)
        assert ws.stop <= ws_bytes and not ws_used[ws].any()
        ws_used[ws] = True
        b = (x.transpose(1, 2, 0) * np.asarray(std, np.float32).reshape(3) + np.asarray(mean, np.float32).reshape(3))
        b = b * np.float32(255)
        back = numpy_u8(np.where(b < 0, np.float32(0), np.where(b > 255, np.float32(255), b)))
        for view, (ptr, c, col) in enumerate([(e["hm"], 1, colors[:1]), (e["hm_hp"], C, colors[1:1 + C])]):
            prod = read(int(ptr), c * h * w).reshape(c, h, w)[:, :, :, None] * col[:, None, None, :]
            m = prod[0]
            for q in prod[1:]:
                m = np.where(np.isnan(q) | (~np.isnan(m) & (q > m)), q, m)
            fore = resize_linear(numpy_u8(m), h * dr, w * dr)
            if theme == "white":
                fore = 255 - fore
            if fore.shape[:2] != (H, W):
                fore = resize_linear(fore, W, H)
            v = back.astype(np.float64) * (1.0 - 0.7) + fore.astype(np.float64) * 0.7
            o = slice(int(e["out_offset"]) + view * H * W * 3, int(e["out_offset"]) + (view + 1) * H * W * 3)
            assert o.stop <= out_bytes and not out_used[o].any()
            out_used[o] = True
            out[o] = np.minimum(v, 255).astype(np.uint8).reshape(-1)
    return out


def test_oracle_equals_golden():
    cases, mean, std = golden_cases()
    for x, hm, hp, dr, want in cases:
        for theme in THEMES:
            got = heatmaps_ref.heatmap_views(x, hm, hp, dr, theme, mean, std)
            for v in heatmaps.VIEWS:
                assert np.array_equal(got[v], want[theme][v]), (x.shape, hp.shape, theme, v)


def test_golden_covers_the_cases():
    cases, mean, std = golden_cases()
    shapes = {hp.shape[1:] for _, _, hp, _, _ in cases}
    assert {(8, 40), (40, 8), (1, 1)} <= shapes
    assert any(h > w for h, w in shapes) and any(h < w for h, w in shapes) and any(h == w > 1 for h, w in shapes)
    assert {dr for _, _, _, dr, _ in cases} == {2, 4} and {hp.shape[0] for _, _, hp, _, _ in cases} == {3, 17}
    maps = np.concatenate([np.concatenate([hm.reshape(-1), hp.reshape(-1)]) for _, hm, hp, _, _ in cases])
    assert (maps == 0).any() and (maps == 1).any() and (maps < 0).any() and (maps > 1).any()
    on = np.float32(np.arange(256) / 255)
    assert np.isin(on, maps).sum() > 200 and np.isin(np.nextafter(on[1:], np.float32(0)), maps).sum() > 200
    backs = [heatmaps_ref.back_image(x, mean, std) for x, _, _, _, _ in cases]
    assert any((b == 0).any() and (b == 255).any() for b in backs)
    # the float32 round trip of a uint8 value through the normalization lands just below it and truncates
    for x, _, _, _, _ in cases[:1]:
        b = (x * std.reshape(3, 1, 1) + mean.reshape(3, 1, 1)) * np.float32(255)
        assert ((np.rint(b) - b > 0) & (np.rint(b) - b < 1e-3)).sum() > 100


@pytest.mark.parametrize("theme", THEMES)
def test_layout_replays_to_the_oracle(theme):
    """Two flip-test batches of different sizes in one table, every other image of each; NaN and out-of-range map
    values and inputs that de-normalize outside [0, 255]."""
    rng = np.random.default_rng(9)
    mean, std = np.array([0.408, 0.447, 0.470], np.float32), np.array([0.289, 0.274, 0.278], np.float32)
    groups = []
    for B, h, w, C in [(3, 6, 10, 17), (2, 9, 9, 5)]:
        x = torch.from_numpy(rng.normal(0, 3, (2 * B, 3, 4 * h, 4 * w)).astype(np.float32))
        hm = torch.from_numpy(rng.random((2 * B, 1, h, w)).astype(np.float32))
        hp = torch.from_numpy(rng.normal(0.5, 2, (2 * B, C, h, w)).astype(np.float32))
        hp[0, 1, 0, 0] = float("nan")
        hp[0, 2, 1, 1] = 3e9
        groups.append((B, x, hm, hp))
    sources, sizes, want = [], [], []
    for B, x, hm, hp in groups:
        for b in range(0, 2 * B, 2):
            sources.append((x[b].data_ptr(), hm[b].data_ptr(), hp[b].data_ptr()))
            sizes.append((x.shape[2], x.shape[3], hm.shape[2], hm.shape[3], hp.shape[1]))
            want.append(heatmaps_ref.heatmap_views(x[b].numpy(), hm[b].numpy(), hp[b].numpy(), 4, theme, mean, std))
    table, offsets, ws = heatmaps.layout(sources, sizes, 4)
    assert table.dtype.itemsize == 64 and offsets[0] == 0
    bases = [t for _, x, hm, hp in groups for t in (x, hm, hp)]
    out_bytes = offsets[-1] + heatmaps.view_bytes(*sizes[-1][:2])
    out = replay(table, bases, out_bytes, ws, theme, mean, std)
    for o, (H, W, _, _, _), w in zip(offsets, sizes, want):
        for k, v in enumerate(heatmaps.VIEWS):
            got = out[o + k * H * W * 3:o + (k + 1) * H * W * 3].reshape(H, W, 3)
            assert np.array_equal(got, w[v]), (H, W, v)


def test_layout_places_views_at_given_offsets():
    sizes = [(8, 12, 2, 3, 17), (4, 4, 1, 1, 1)]
    table, offsets, ws = heatmaps.layout([(16, 32, 64), (128, 256, 512)], sizes, 4, [1000, 0])
    assert offsets == [1000, 0] and table["out_offset"].tolist() == [1000, 0]
    assert table["input"].tolist() == [16, 128] and table["hm_hp"].tolist() == [64, 512]
    assert table["ws_offset"].tolist() == [0, 2 * (6 + 96) * 3 // 16 * 16 + 16]
    assert ws == table["ws_offset"][1] + (2 * (1 + 16) * 3 + 15) // 16 * 16


def _ok(h=3, w=5, C=17, dr=4):
    return [torch.zeros(3, h * dr, w * dr)], [torch.zeros(1, h, w)], [torch.zeros(C, h, w)]


@pytest.mark.parametrize("bad", ["dtype", "contiguous", "rank", "input_c", "hm_c", "c0", "c18", "hp_size", "dr",
                                 "count", "cpu"])
def test_checks_reject_bad_inputs(bad):
    x, hm, hp = _ok()
    dr = 4
    if bad == "dtype":
        hm = [hm[0].double()]
    elif bad == "contiguous":
        x = [torch.zeros(3, 20, 12).transpose(1, 2)]
    elif bad == "rank":
        hp = [hp[0][None]]
    elif bad == "input_c":
        x = [torch.zeros(4, 12, 20)]
    elif bad == "hm_c":
        hm = [torch.zeros(2, 3, 5)]
    elif bad == "c0":
        hp = [torch.zeros(0, 3, 5)]
    elif bad == "c18":
        hp = [torch.zeros(18, 3, 5)]
    elif bad == "hp_size":
        hp = [torch.zeros(17, 5, 3)]
    elif bad == "dr":
        dr = 2
    elif bad == "count":
        hp = hp * 2
    with pytest.raises(ValueError):
        heatmaps.check(x, hm, hp, dr)
    with pytest.raises(ValueError):
        heatmaps.views(x, hm, hp, dr, "white", np.zeros(3), np.ones(3))


def test_checks_reject_too_many_images():
    x, hm, hp = _ok()
    with pytest.raises(ValueError, match="65535"):
        heatmaps.check(x * 65536, hm * 65536, hp * 65536, 4)


def test_numpy_cast_the_kernel_copies():
    v = np.array([-1.5, 300.7, -300, np.nan, np.inf, -np.inf, 2.0 ** 31, -2.0 ** 31, 3e9, -3e9, 255.9, 256, 0.99,
                  -0.99, 2.0 ** 31 - 128, -(2.0 ** 31 - 128)], np.float32)
    with np.errstate(invalid="ignore"):
        cast = v.astype(np.uint8)
    assert cast[:4].tolist() == [255, 44, 212, 0]
    assert np.array_equal(cast, numpy_u8(v))
    rng = np.random.default_rng(1)
    w = np.concatenate([rng.normal(0, s, 20000) for s in (1, 300, 1e5, 1e9, 1e10)]).astype(np.float32)
    with np.errstate(invalid="ignore"):
        assert np.array_equal(w.astype(np.uint8), numpy_u8(w))
        # the max over the colours propagates NaN, as the kernel's select does
        assert np.array_equal(np.stack([w, np.where(w > 0, np.nan, w)]).max(0).astype(np.uint8), numpy_u8(
            np.where(w > 0, np.nan, w)))


def test_colors():
    assert heatmaps.colors("white")[0].tolist() == [255, 128, 128]
    assert heatmaps.colors("black")[0].tolist() == [255, 255, 255]
    assert heatmaps.colors("white").shape == (18, 3) and heatmaps.colors("white").dtype == np.float32
    assert np.array_equal(heatmaps.colors("white")[1:], 255 - heatmaps.colors("black")[1:])
