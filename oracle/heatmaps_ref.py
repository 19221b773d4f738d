"""ORACLE (test infrastructure, not product): numpy / cv2 restatement of the heat-map views the reference's
``MultiPoseDetector.debug`` adds with ``DEBUG >= 2`` (``lib/detectors/multi_pose.py:82-94`` with
``lib/utils/debugger.py`` ``gen_colormap`` / ``gen_colormap_hp`` / ``add_blend_img``), the companion of
``oracle.debugger_ref`` for the drawn poses.  ``tests/golden/heatmap_views.npz`` pins it to the unmodified reference
Debugger (``oracle/make_golden_heatmaps.py``); ``csrc/heatmaps.cu`` is checked against it byte for byte.
"""
from __future__ import annotations

import cv2
import numpy as np

from centerpose_b200.render import JOINT_COLORS, theme_color


def back_image(x, mean, std):
    """The (H, W, 3) uint8 image ``debug()`` blends onto: the normalized (3, H, W) float32 input de-normalized in
    float32 and truncated, so a round trip of 255 that lands on 254.99998 gives 254."""
    img = np.asarray(x, np.float32).transpose(1, 2, 0)
    mean, std = np.asarray(mean, np.float32).reshape(3), np.asarray(std, np.float32).reshape(3)
    with np.errstate(invalid="ignore"):
        return np.clip((img * std + mean) * np.float32(255), 0, 255).astype(np.uint8)


def colormap(maps, colors):
    """max over c of maps[c] * colors[c] in float32 per channel, cast to uint8 as numpy casts (out-of-range values
    wrap, NaN gives 0)."""
    prod = np.asarray(maps, np.float32)[:, :, :, None] * np.asarray(colors, np.float32)[:len(maps), None, None, :]
    with np.errstate(invalid="ignore"):
        return prod.max(axis=0).astype(np.uint8)


def fore_image(maps, colors, dr, theme, H, W):
    """The (H, W, 3) uint8 image blended onto the input: the colour map resized to (h * dr, w * dr) (width h * dr),
    inverted with the 'white' theme, then resized to (W, H) unless its row count equals both H and W."""
    _, h, w = maps.shape
    fore = cv2.resize(colormap(maps, colors), (h * dr, w * dr))
    if theme == "white":
        fore = 255 - fore
    if fore.shape[0] != H or fore.shape[0] != W:
        fore = cv2.resize(fore, (W, H))
    return fore


def blend_view(back, maps, colors, dr, theme):
    """One view: ``fore_image`` blended onto ``back`` 0.3 / 0.7 in float64."""
    fore = fore_image(maps, colors, dr, theme, *back.shape[:2])
    return np.clip(back * (1. - 0.7) + fore * 0.7, 0, 255).astype(np.uint8)


def map_colors(theme):
    """The (1, 3) hm colour and the (17, 3) joint colours, float32, with the theme applied."""
    hp = np.array(JOINT_COLORS, np.float32)
    if theme == "white":
        hp = 255 - hp
    return np.array([theme_color(theme)], np.float32), hp


def heatmap_views(x, hm, hm_hp, dr, theme, mean, std):
    """``{'pred_hm', 'pred_hmhp'}`` for one image: ``x`` its (3, H, W) normalized input, ``hm`` its (1, h, w) and
    ``hm_hp`` its (C, h, w) maps as ``process()`` leaves them (numpy arrays)."""
    back = back_image(x, mean, std)
    hm_color, hp_colors = map_colors(theme)
    return {"pred_hm": blend_view(back, np.asarray(hm), hm_color, dr, theme),
            "pred_hmhp": blend_view(back, np.asarray(hm_hp), hp_colors, dr, theme)}
