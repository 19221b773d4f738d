"""ORACLE (test infrastructure, not product): numpy restatement of the reference's
``multi_pose_decode`` and its helpers, float32 arithmetic in the reference's order.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline /
``--impl reference`` legs may import this module.  The product path
(``centerpose_b200``) never does.

Follows (``/root/reference``):
  * ``lib/models/decode.py:10-16``   ``_nms``            -> :func:`nms3x3`
  * ``lib/models/decode.py:87-96``   ``_topk_channel``   -> :func:`topk_channel`
  * ``lib/models/decode.py:99-115``  ``_topk``           -> :func:`topk`
  * ``lib/models/utils.py:11-25``    ``_gather_feat`` / ``_transpose_and_gather_feat``
                                                          -> :func:`gather_nchw`
  * ``lib/models/decode.py:235-308`` ``multi_pose_decode`` -> :func:`multi_pose_decode`

Pinning: the reference has no golden vectors for this path (SURVEY.md §4, §8c), so this
restatement is pinned by running the reference's own Python here
(``oracle/make_golden.py``) and committing its outputs under ``tests/golden/``;
``tests/test_oracle_golden.py`` replays them.

Ties: ``torch.topk`` / ``min(dim)`` leave tie order implementation-defined in the
reference.  The oracle fixes the canonical order (value descending, flat index
ascending; first minimum) — the same rule the CUDA kernel implements — and the golden
inputs are tie-free so both agree with the reference exactly.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def nms3x3(heat: np.ndarray) -> np.ndarray:
    """decode.py:10-16 — 3x3/s1/p1 max-pool (implicit -inf padding), keep cells equal to
    their window max, zero the rest (``heat * keep``)."""
    heat = np.asarray(heat, dtype=F32)
    B, C, H, W = heat.shape
    pad = np.full((B, C, H + 2, W + 2), -np.inf, dtype=F32)
    pad[:, :, 1:-1, 1:-1] = heat
    hmax = pad[:, :, 1:-1, 1:-1].copy()
    for dy in (0, 1, 2):
        for dx in (0, 1, 2):
            np.maximum(hmax, pad[:, :, dy:dy + H, dx:dx + W], out=hmax)
    keep = (hmax == heat).astype(F32)
    return heat * keep


def _topk_lastdim(flat: np.ndarray, K: int):
    """top-K along the last axis, sorted descending, ties -> lower index first."""
    order = np.argsort(-flat, axis=-1, kind="stable")[..., :K]
    vals = np.take_along_axis(flat, order, axis=-1)
    return vals, order.astype(np.int64)


def topk_channel(scores: np.ndarray, K: int):
    """decode.py:87-96 — per (batch, channel) top-K over H*W."""
    B, C, H, W = scores.shape
    if K > H * W:
        raise RuntimeError("selected index k out of range")  # what torch.topk raises
    vals, inds = _topk_lastdim(scores.reshape(B, C, H * W), K)
    inds = inds % (H * W)
    ys = (inds // W).astype(F32)   # (ind / width).int().float()
    xs = (inds % W).astype(F32)
    return vals, inds, ys, xs


def topk(scores: np.ndarray, K: int):
    """decode.py:99-115 — per-class top-K then a cross-class top-K over C*K."""
    B, C, H, W = scores.shape
    vals, inds, ys, xs = topk_channel(scores, K)
    score, ind = _topk_lastdim(vals.reshape(B, C * K), K)
    clses = (ind // K).astype(np.int32)
    inds = np.take_along_axis(inds.reshape(B, C * K), ind, axis=1)
    ys = np.take_along_axis(ys.reshape(B, C * K), ind, axis=1)
    xs = np.take_along_axis(xs.reshape(B, C * K), ind, axis=1)
    return score, inds, clses, ys, xs


def gather_nchw(feat: np.ndarray, ind: np.ndarray) -> np.ndarray:
    """utils.py:11-25 — feat (B,C,H,W), ind (B,N) flat cell indices -> (B,N,C).
    (The reference materialises the NHWC transpose first; the values are identical.)"""
    B, C, H, W = feat.shape
    flat = feat.reshape(B, C, H * W)
    out = np.take_along_axis(flat, ind[:, None, :].astype(np.int64), axis=2)  # (B,C,N)
    return np.ascontiguousarray(out.transpose(0, 2, 1))


def multi_pose_decode(heat, wh, kps, reg=None, hm_hp=None, hp_offset=None, K=100):
    """decode.py:235-308.  Inputs fp32 NCHW; ``heat``/``hm_hp`` already sigmoid'ed.
    Returns (B, K, 4+1+2J+J) float32: [x1,y1,x2,y2, score, J*(x,y), J*kp_score]."""
    heat = np.asarray(heat, F32); wh = np.asarray(wh, F32); kps = np.asarray(kps, F32)
    B, cat, H, W = heat.shape
    J = kps.shape[1] // 2
    heat = nms3x3(heat)                                              # :241
    scores, inds, clses, ys, xs = topk(heat, K)                      # :242
    kps_g = gather_nchw(kps, inds).reshape(B, K, J * 2).copy()       # :244-245
    kps_g[..., 0::2] += xs[:, :, None]                               # :246
    kps_g[..., 1::2] += ys[:, :, None]                               # :247
    if reg is not None:                                              # :248-252
        reg_g = gather_nchw(np.asarray(reg, F32), inds)
        xs = xs[:, :, None] + reg_g[:, :, 0:1]
        ys = ys[:, :, None] + reg_g[:, :, 1:2]
    else:                                                            # :253-255
        xs = xs[:, :, None] + F32(0.5)
        ys = ys[:, :, None] + F32(0.5)
    wh_g = gather_nchw(wh, inds)                                     # :256-257
    scores = scores[:, :, None]
    bboxes = np.concatenate([xs - wh_g[..., 0:1] / F32(2), ys - wh_g[..., 1:2] / F32(2),
                             xs + wh_g[..., 0:1] / F32(2), ys + wh_g[..., 1:2] / F32(2)],
                            axis=2).astype(F32)                      # :261-264
    if hm_hp is None:
        # decode.py:307 references hm_score unconditionally -> NameError in the reference.
        raise NameError("name 'hm_score' is not defined")
    hm_hp = nms3x3(np.asarray(hm_hp, F32))                           # :266
    thresh = F32(0.1)                                                # :267
    kps_j = kps_g.reshape(B, K, J, 2).transpose(0, 2, 1, 3)          # b x J x K x 2  :268-269
    hm_score, hm_inds, hm_ys, hm_xs = topk_channel(hm_hp, K)         # b x J x K      :271
    if hp_offset is not None:                                        # :272-277
        off = gather_nchw(np.asarray(hp_offset, F32), hm_inds.reshape(B, -1)).reshape(B, J, K, 2)
        hm_xs = hm_xs + off[..., 0]
        hm_ys = hm_ys + off[..., 1]
    else:                                                            # :278-280
        hm_xs = hm_xs + F32(0.5)
        hm_ys = hm_ys + F32(0.5)
    mask = (hm_score > thresh).astype(F32)                           # :282
    hm_score = (F32(1) - mask) * F32(-1) + mask * hm_score           # :283
    hm_ys = (F32(1) - mask) * F32(-10000) + mask * hm_ys             # :284
    hm_xs = (F32(1) - mask) * F32(-10000) + mask * hm_xs             # :285
    # :286-289  dist[b,j,p,c] = sqrt((kx[p]-hx[c])^2 + (ky[p]-hy[c])^2), fp32, no FMA
    dx = kps_j[..., 0][:, :, :, None] - hm_xs[:, :, None, :]
    dy = kps_j[..., 1][:, :, :, None] - hm_ys[:, :, None, :]
    dist = np.sqrt((dx * dx).astype(F32) + (dy * dy).astype(F32)).astype(F32)
    min_ind = np.argmin(dist, axis=3)                                # first minimum
    min_dist = np.take_along_axis(dist, min_ind[..., None], axis=3)  # b x J x K x 1
    sel_score = np.take_along_axis(hm_score, min_ind, axis=2)[..., None]   # :290
    sel_x = np.take_along_axis(hm_xs, min_ind, axis=2)[..., None]    # :292-295
    sel_y = np.take_along_axis(hm_ys, min_ind, axis=2)[..., None]
    l = bboxes[:, None, :, 0:1]; t = bboxes[:, None, :, 1:2]         # :296-299
    r = bboxes[:, None, :, 2:3]; b = bboxes[:, None, :, 3:4]
    rej = ((sel_x < l) | (sel_x > r) | (sel_y < t) | (sel_y > b) | (sel_score < thresh) |
           (min_dist > (np.maximum(b - t, r - l) * F32(0.3))))       # :300-302
    rej = rej.astype(F32)
    out_x = (F32(1) - rej) * sel_x + rej * kps_j[..., 0:1]           # :304
    out_y = (F32(1) - rej) * sel_y + rej * kps_j[..., 1:2]
    kps_out = np.concatenate([out_x, out_y], axis=3).transpose(0, 2, 1, 3).reshape(B, K, J * 2)
    det = np.concatenate([bboxes, scores, kps_out,
                          sel_score[..., 0].transpose(0, 2, 1)], axis=2)  # :306
    return det.astype(F32)


def canonical_rows(det: np.ndarray, inds_hint=None):
    """Sort helper for tie-insensitive comparison: returns rows ordered by
    (score desc, x1, y1) so two decoders that break exact score ties differently
    can still be compared row by row."""
    out = np.empty_like(det)
    for b in range(det.shape[0]):
        d = det[b]
        order = np.lexsort((d[:, 1], d[:, 0], -d[:, 4]))
        out[b] = d[order]
    return out


def synth_decode_inputs(B, H, W, seed=317, J=17, kind="smooth", dtype=F32):
    """Synthetic decode inputs (SURVEY.md §8d "decode kernel alone").

    kind: 'smooth'  sigmoid(2*N(0,1)-2.19) box-filtered 3x3 (realistic peak density)
          'uniform' U(0,1) (adversarial: ~1/9 of cells are local maxima)
          'sparse'  fewer than K positive peaks (zeros get selected)
          'plateau' constant heat-map (every cell ties)
          'lowhp'   all hm_hp <= 0.1 (every joint falls back; col 39+j = -1)
          'sqrttie', 'sqrttie_swap', 'sqtie', 'thresh'
                    constructed tie and threshold cases of the keypoint grouping, see :func:`_constructed`
    Returns dict of fp32 NCHW arrays: heat, wh, kps, reg, hm_hp, hp_offset."""
    if kind in CONSTRUCTED:
        return _constructed(B, H, W, seed, J, kind)
    rng = np.random.RandomState(seed)

    def heatmap(C):
        if kind == "uniform":
            return rng.uniform(0.0, 1.0, size=(B, C, H, W)).astype(F32)
        if kind == "plateau":
            return np.full((B, C, H, W), 0.25, dtype=F32)
        if kind == "sparse":
            h = np.zeros((B, C, H, W), dtype=F32)
            n = max(1, min(37, H * W // 16))
            for b in range(B):
                for c in range(C):
                    ys = rng.randint(0, H, size=n); xs = rng.randint(0, W, size=n)
                    h[b, c, ys, xs] = rng.uniform(0.15, 0.99, size=n).astype(F32)
            return h
        z = (2.0 * rng.randn(B, C, H + 2, W + 2) - 2.19).astype(F32)
        s = (1.0 / (1.0 + np.exp(-z))).astype(F32)
        acc = np.zeros((B, C, H, W), dtype=F32)
        for dy in (0, 1, 2):
            for dx in (0, 1, 2):
                acc += s[:, :, dy:dy + H, dx:dx + W]
        h = (acc / F32(9)).astype(F32)
        if kind == "lowhp":
            h = (h * F32(0.09) / max(float(h.max()), 1e-6)).astype(F32)
        return h

    heat = heatmap(1) if kind != "lowhp" else synth_decode_inputs(B, H, W, seed + 1, J, "smooth")["heat"]
    hm_hp = heatmap(J)
    return dict(
        heat=heat.astype(dtype),
        wh=rng.uniform(0, 40, size=(B, 2, H, W)).astype(dtype),
        kps=(10.0 * rng.randn(B, 2 * J, H, W)).astype(dtype),
        reg=rng.uniform(0, 1, size=(B, 2, H, W)).astype(dtype),
        hm_hp=hm_hp.astype(dtype),
        hp_offset=rng.uniform(0, 1, size=(B, 2, H, W)).astype(dtype),
    )


CONSTRUCTED = ("sqrttie", "sqrttie_swap", "sqtie", "thresh")


def _constructed(B, H, W, seed, J, kind):
    """Hand-placed keypoint-grouping cases on a 'smooth' base whose heat maps are cleared (every image the same;
    needs H, W >= 40).  All placed values are exact fp32.

    'sqrttie'       one person at cell (20,20), joint-0 guess (20.3, 20.0).  Candidate A at cell (20,22), score 0.5,
                    lands at (22.783405, 20.632195); candidate B at cell (20,18), score 0.6, at (17.816463, 20.631685).
                    Their squared distances 6.5669756 (A) and 6.566976 (B) are adjacent floats with the same fp32
                    sqrt: the reference's dist.min() takes B, the first of its score-sorted list.
    'sqrttie_swap'  the same with the scores swapped: A (0.6, the higher flat index) is first in score order.
    'sqtie'         exactly equal squared distances (dx = +-2 on joint 0, dy = +-2 on joint 1): the higher score
                    wins, on joint 0 from the higher flat index, on joint 1 from the lower one.
    'thresh'        four people; on every joint each person has a candidate of exactly fp32(0.1) two cells from its
                    guess (masked: the reference keeps scores > 0.1) and one of nextafter(0.1, 1) four rows away
                    (kept, and within 0.3 * box size), each an isolated 3x3 maximum.  Joint J-1 has only the 0.1
                    candidates, so it has no candidate at all.
    """
    assert H >= 40 and W >= 40, "constructed decode kinds need a map of at least 40x40"
    d = synth_decode_inputs(B, H, W, seed, J, "smooth")
    heat, hm_hp, wh, kps, reg, off = d["heat"], d["hm_hp"], d["wh"], d["kps"], d["reg"], d["hp_offset"]
    heat[:] = 0
    hm_hp[:] = 0
    f = F32
    if kind in ("sqrttie", "sqrttie_swap"):
        sa, sb = (f(0.5), f(0.6)) if kind == "sqrttie" else (f(0.6), f(0.5))
        heat[:, 0, 20, 20] = f(0.9)
        wh[:, :, 20, 20] = f(30)
        kps[:, 0, 20, 20] = f(0.3); kps[:, 1, 20, 20] = f(0.0)
        hm_hp[:, 0, 20, 22] = sa; off[:, 0, 20, 22] = f(0.7834044); off[:, 1, 20, 22] = f(0.6321947)
        hm_hp[:, 0, 20, 18] = sb; off[:, 0, 20, 18] = f(-0.18353653); off[:, 1, 20, 18] = f(0.63168526)
    elif kind == "sqtie":
        heat[:, 0, 20, 20] = f(0.9)
        wh[:, :, 20, 20] = f(30)
        kps[:, 0:2, 20, 20] = (f(0.5), f(0.0))            # joint 0 guess (20.5, 20.0)
        hm_hp[:, 0, 20, 18] = f(0.5); off[:, :, 20, 18] = (f(0.5), f(0.0))      # (18.5, 20.0)
        hm_hp[:, 0, 20, 23] = f(0.6); off[:, :, 20, 23] = (f(-0.5), f(0.0))     # (22.5, 20.0)
        kps[:, 2:4, 20, 20] = (f(0.0), f(0.5))            # joint 1 guess (20.0, 20.5)
        hm_hp[:, 1, 18, 20] = f(0.7); off[:, :, 18, 20] = (f(0.0), f(0.5))      # (20.0, 18.5)
        hm_hp[:, 1, 23, 20] = f(0.4); off[:, :, 23, 20] = (f(0.0), f(-0.5))     # (20.0, 22.5)
    elif kind == "thresh":
        t, t_up = f(0.1), np.nextafter(f(0.1), f(1))
        for (y, x), s in zip(((8, 8), (8, 28), (26, 8), (26, 28)), (0.9, 0.8, 0.7, 0.6)):
            heat[:, 0, y, x] = f(s)
            wh[:, :, y, x] = f(16); reg[:, :, y, x] = f(0.5)
            kps[:, :, y, x] = 0                            # every joint's guess is the cell (x, y)
            hm_hp[:, :, y, x + 2] = t; off[:, :, y, x + 2] = f(0.5)       # (x + 2.5, y + 0.5): masked
            hm_hp[:, :J - 1, y + 4, x] = t_up; off[:, :, y + 4, x] = f(0.5)   # (x + 0.5, y + 4.5): kept
    return d
