"""CPU tests of the device resize's arithmetic and of run_images' upload layout.

``resize_linear`` is the integer model of ``cv2.resize(img, (new_w, new_h))`` (INTER_LINEAR, uint8) that
``cpb200_resize_linear_u8_batch`` (csrc/post.cu) implements; here it is pinned against the installed OpenCV on a grid
of sizes and scales, upscales included.  ``pack_group`` is checked by replaying the kernels' table reads on the host."""
import itertools

import cv2
import numpy as np
import pytest
import torch

SCALES = [0.5, 0.75, 1.25, 1.5, 2, 0.7, 1.1]          # 0.7 and 1.1: int(h * scale) truncates for most sizes
SIZES = [(480, 640), (427, 640), (640, 427), (333, 500), (37, 51), (33, 17), (9, 1), (1, 9), (1, 1), (5, 3), (7, 4),
         (2, 3), (4, 4)]


def _taps(d, n_in, n_out):
    """Source index and 11-bit weight of the first tap per output coordinate (resize.cpp, resizeGeneric_)."""
    f = ((d + 0.5) * (1.0 / (n_out / n_in)) - 0.5).astype(np.float32)
    i = np.floor(f)
    f = (f - i).astype(np.float32)
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    return i.astype(np.int64), a0


def resize_linear(img, new_w, new_h):
    h, w, _ = img.shape
    xi, a0 = _taps(np.arange(new_w), w, new_w)
    clamp = (xi < 0) | (xi >= w - 1)                   # columns: the coefficient is clamped at the border
    xi, a0 = np.clip(xi, 0, w - 1), np.where(clamp, 2048, a0)
    yi, b0 = _taps(np.arange(new_h), h, new_h)         # rows: the weights stay, each source row is clipped on its own
    s = img.astype(np.int64)
    hz = s[:, xi] * a0[None, :, None] + s[:, np.minimum(xi + 1, w - 1)] * (2048 - a0)[None, :, None]
    h0, h1 = hz[np.clip(yi, 0, h - 1)], hz[np.clip(yi + 1, 0, h - 1)]
    t = ((h0 >> 4) * b0[:, None, None] >> 16) + ((h1 >> 4) * (2048 - b0)[:, None, None] >> 16)
    return np.clip((t + 2) >> 2, 0, 255).astype(np.uint8)


def _grid():
    for (h, w), scale in itertools.product(SIZES, SCALES):
        if int(h * scale) >= 1 and int(w * scale) >= 1:
            yield h, w, scale


@pytest.mark.parametrize("scale", SCALES)
def test_resize_model_equals_cv2(scale):
    rng = np.random.RandomState(int(scale * 100))
    cases = [(h, w) for h, w, s in _grid() if s == scale]
    assert len(cases) >= 8
    for h, w in cases:
        for img in (rng.randint(0, 256, (h, w, 3)).astype(np.uint8),
                    np.where(rng.rand(h, w, 3) < 0.5, 0, 255).astype(np.uint8)):      # extreme values, no saturation
            new_h, new_w = int(h * scale), int(w * scale)
            want = cv2.resize(img, (new_w, new_h))
            got = resize_linear(img, new_w, new_h)
            assert got.shape == want.shape and np.array_equal(got, want), ((h, w), scale, int((got != want).sum()))


def _replay(buf, at, images):
    """What the device does with one packed group: resize each image through the resize table (the model above),
    then read each pre-process input through the pre-process table."""
    from centerpose_b200.detector import _PRE_IMAGE, _RESIZE_IMAGE
    B = len(images)
    pixels = buf[at["o_img"]:]
    if at["o_rsz"] is not None:
        scratch = np.zeros(at["scratch"], np.uint8)
        for e in buf[at["o_rsz"]:at["o_rsz"] + B * 32].view(_RESIZE_IMAGE):
            src = pixels[e["src_offset"]:e["src_offset"] + e["h"] * e["w"] * 3].reshape(e["h"], e["w"], 3)
            out = resize_linear(src, int(e["new_w"]), int(e["new_h"])).reshape(-1)
            assert 0 <= e["dst_offset"] and e["dst_offset"] + out.size <= scratch.size
            scratch[e["dst_offset"]:e["dst_offset"] + out.size] = out
        pixels = scratch
    pre = buf[:B * 64].view(_PRE_IMAGE)
    return [pixels[e["offset"]:e["offset"] + e["h"] * e["w"] * 3].reshape(e["h"], e["w"], 3) for e in pre], pre


@pytest.mark.parametrize("scale", [1, 0.75, 2])
def test_pack_group_layout(scale):
    from centerpose_b200.detector import pack_group
    rng = np.random.RandomState(5)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(48, 64), (37, 51), (64, 48), (2, 9)]]
    new_shapes = [(int(im.shape[0] * scale), int(im.shape[1] * scale)) for im in images]
    trans = [rng.randn(2, 3) for _ in images]
    aff = rng.randn(len(images), 6).astype(np.float32)
    dst = [7, 0, 3, 3]
    buf, at = pack_group(images, new_shapes, trans, aff, dst, alloc=lambda n: torch.empty(n, dtype=torch.uint8))
    hv = buf.numpy()
    assert at["o_img"] % 16 == 0 and at["o_idx"] % 8 == 0 and at["o_aff"] % 8 == 0
    assert hv.size == at["o_img"] + sum(im.nbytes for im in images)
    np.testing.assert_array_equal(hv[at["o_aff"]:at["o_idx"]].view(np.float32).reshape(-1, 6), aff)
    assert hv[at["o_idx"]:at["o_idx"] + 8 * len(images)].view(np.int64).tolist() == dst
    if scale == 1:
        assert at["o_rsz"] is None and at["scratch"] == 0 and at["o_aff"] == 64 * len(images)
    else:
        # the pinned buffer carries the raw pixels; the scaled images exist only in the scratch buffer
        assert at["o_rsz"] == 64 * len(images) and at["o_aff"] == 96 * len(images)
        assert at["scratch"] == sum(h * w * 3 for h, w in new_shapes)
    inputs, pre = _replay(hv, at, images)
    for n, im in enumerate(images):
        want = im if scale == 1 else cv2.resize(im, new_shapes[n][::-1])
        assert np.array_equal(inputs[n], want), n
        np.testing.assert_array_equal(pre[n]["trans_input"], trans[n].reshape(6))


def test_pack_group_resizes_a_mixed_group_and_rejects_empty_sizes():
    """One image keeps its size in a group where another changes: both go through the resize (an identity for the
    first, as cv2.resize to the same size is a copy).  Sizes below 1 never reach the device."""
    from centerpose_b200.detector import pack_group, resize_table
    rng = np.random.RandomState(6)
    images = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(3, 4), (30, 40)]]
    new_shapes = [(3, 4), (31, 41)]
    buf, at = pack_group(images, new_shapes, [np.eye(2, 3)] * 2, np.zeros((2, 6), np.float32), [0, 1])
    assert at["o_rsz"] is not None
    inputs, _ = _replay(buf, at, images)
    assert np.array_equal(inputs[0], images[0]) and np.array_equal(inputs[1], cv2.resize(images[1], (41, 31)))
    for bad in ([(0, 4)], [(3, 0)]):
        with pytest.raises(ValueError):
            resize_table([(3, 4)], bad)
        with pytest.raises(ValueError):
            pack_group(images[:1], bad, [np.eye(2, 3)], np.zeros((1, 6), np.float32), [0])
    with pytest.raises(ValueError):
        resize_table([(0, 4)], [(3, 4)])
