"""Constructed inputs of the fused decode kernel (tests/test_decode_cases_gpu.py, tests/test_decode_cases_cpu.py).
A helper module: it holds no tests.

Random maps reach the common path of ``csrc/decode.cu`` and some fallbacks by accident.  ``CASES`` places every peak
where one branch of the kernel needs it: on the strip, float4 and warp seams of the three phase-1 scans, past one warp's
512-candidate segment, into each outcome of the adaptive bucket select, into the centre-list fill, onto the keypoint
threshold and into every tie of the keypoint grouping.  Each case names the branches (``BRANCHES``) it is built to reach.

The second half of the module restates the kernel's own control arithmetic on the numpy maps (which scan runs, which
warp segment a cell's peak goes to and in what order, the bucket select's histogram rounds, the grouping's ties), so
that ``reached(case)`` can show from the data alone that a case reaches what it claims.  Every placed value is exact
fp32.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, FrozenSet

import numpy as np

from oracle import decode_ref

F32 = np.float32
TPB, CAP, SEG, BND, MAXK, MAXJ = 256, 4096, 512, 64, 128, 32     # decode.cu constants, CPB200_DECODE_MAX_K / _J
THRESH = F32(0.1)

BRANCHES = {
    "scan_w128": "scan_w128: W == 128, H % 8 == 0, 16-byte aligned map (one warp per row strip)",
    "scan_vec": "scan_vec: W % 4 == 0, aligned, not the W == 128 specialisation",
    "scan_vec_shared_warp": "scan_vec with W / 4 column groups not a multiple of 32: one warp spans several strips",
    "scan_vec_two_pass": "scan_vec with more than 256 column groups: each thread takes two column groups",
    "scan_scalar": "scan_scalar: W % 4 != 0",
    "scan_scalar_misaligned": "scan_scalar on a map that is not 16-byte aligned (W % 4 == 0)",
    "seam_strip": "a peak on the first or last row of a row strip (read through the next strip's halo row)",
    "seam_float4": "a peak on column 4g-1 or 4g (its neighbour is in another thread's float4)",
    "seam_warp": "a peak whose neighbour belongs to another warp (lane 31 | lane 0, or another strip's warp)",
    "seam_corner": "peaks on all four corners of the map",
    "seam_plateau": "two equal neighbouring peaks owned by different threads: both are kept",
    "count_eq_k": "centre map with exactly K candidates",
    "count_k_plus_1": "centre map with exactly K + 1 candidates",
    "segment_overflow": "one warp segment holds more than 512 candidates while the map holds at most 4096",
    "centre:bucket_take_whole": "centre: the boundary bucket is exactly what is still needed",
    "centre:bucket_resolve_ties": "centre: 2..64 keys in the boundary bucket, exact ties at the K-th value",
    "centre:bucket_refine": "centre: more than 64 keys in the first boundary bucket, resolved after narrowing",
    "centre:bucket_give_up": "centre: more than 64 exact ties at the K-th value -> select_slow",
    "centre:bucket_max_rounds": "centre: a subnormal-to-1 value span that needs four histogram rounds",
    "joint:bucket_take_whole": "joint: the boundary bucket is exactly what is still needed",
    "joint:bucket_resolve_ties": "joint: 2..64 keys in the boundary bucket, exact ties at the K-th value",
    "joint:bucket_refine": "joint: more than 64 keys in the first boundary bucket, resolved after narrowing",
    "joint:bucket_give_up": "joint: more than 64 exact ties at the K-th value -> select_slow",
    "fill_n_ge_2k": "fewer than K positive centre peaks, H*W >= 2K",
    "fill_n_lt_2k": "fewer than K positive centre peaks, H*W < 2K",
    "fill_all_zero": "an all-zero centre map",
    "fill_neg_zero": "-0.0 cells in a centre map with fewer than K peaks",
    "fill_negative_peak": "fewer than K positive centre peaks and a negative peak -> select_slow",
    "mask_exact_thresh": "isolated keypoint peaks of exactly fp32(0.1) (masked) and nextafter(0.1, 1) (kept)",
    "mask_no_candidate": "a joint with no candidate above 0.1",
    "mask_over_k_ties": "a joint with more than K candidates above 0.1 and exact ties at the K-th",
    "group_sqrt_tie": "two candidates with equal fp32 sqrt distance and different squared distances; the first in "
                      "score order has the larger squared distance",
    "group_sqrt_tie_swapped": "the same with the first in score order at the smaller squared distance and the higher "
                              "flat index",
    "group_sq_tie_score": "exactly equal squared distances, different scores: the higher score wins",
    "group_sq_tie_index": "exactly equal squared distances and scores: the lower flat index wins",
    "group_tie_across_halves": "K odd, the tied candidates on both sides of the half-CTA split (K + 1) / 2",
    "group_box_edge": "the chosen candidate exactly on a box edge (kept: the tests are < and >)",
    "group_min_dist_edge": "min_dist exactly 0.3 * max(h, w) (kept)",
    "group_k1": "K == 1",
    "group_no_reg_off": "reg and hp_offset both None",
    "batch_many_ctas": "B = 48, J = 17: 864 CTAs, more than are resident at once, every image different",
    "joints_1": "J == 1",
    "joints_32": "J == 32 (CPB200_DECODE_MAX_J)",
}


@dataclass
class Inputs:
    maps: Dict[str, np.ndarray]            # heat, wh, kps, reg, hm_hp, hp_offset: fp32 NCHW
    K: int
    use_reg: bool = True
    use_off: bool = True
    misaligned: bool = False               # run from a contiguous view one float past a 16-byte boundary

    @property
    def shape(self):
        B, _, H, W = self.maps["heat"].shape
        return B, H, W, self.maps["hm_hp"].shape[1]


@dataclass(frozen=True)
class DecodeCase:
    name: str
    build: Callable[[], Inputs]
    reason: str
    branches: FrozenSet[str] = field(default_factory=frozenset)


CASES = []


def add(name, build, reason, *branches):
    assert all(b in BRANCHES for b in branches), [b for b in branches if b not in BRANCHES]
    CASES.append(DecodeCase(name, build, reason, frozenset(branches)))


# ------------------------------------------------------------------------------------------- the kernel's arithmetic
def scan_route(H, W, aligned=True):
    """decode_kernel's phase-1 dispatch"""
    if aligned and W % 4 == 0:
        return "w128" if (W == 128 and H % 8 == 0) else "vec"
    return "scalar"


def owners(H, W, route):
    """per cell: (thread u of the scan, warp, strip, column group) as the scan assigns them; strip / group are -1 on the
    scalar path.  scan_vec: XG = W/4 groups, S = clamp(256 / XG, 1, H) strips of RS = ceil(H / S) rows, u = st*XG + g;
    scan_w128 is the same arithmetic with XG = 32, S = 8.  scan_scalar: u = the flat cell index."""
    y, x = np.mgrid[0:H, 0:W]
    if route == "scalar":
        u = y * W + x
        return dict(u=u, warp=(u % TPB) // 32, lane=u % 32, pas=u // TPB, row=np.zeros_like(u),
                    strip=np.full_like(u, -1), group=np.full_like(u, -1))
    XG = W // 4
    S = min(max(TPB // XG, 1), H)
    RS = -(-H // S)
    st, g = y // RS, x // 4
    u = st * XG + g
    return dict(u=u, warp=(u % TPB) // 32, lane=u % 32, pas=u // TPB, row=y - st * RS, strip=st, group=g)


def peak_mask(m):
    """cells equal to their 3x3 window max (implicit -inf padding): the kernel's '==' NMS rule"""
    H, W = m.shape
    pad = np.full((H + 2, W + 2), -np.inf, F32)
    pad[1:-1, 1:-1] = m
    mx = np.max(np.stack([pad[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)]), axis=0)
    return mx == m


def candidates(m, floor, route):
    """(values, flat indices) of the peaks above ``floor`` in the order compact_segments leaves them (warp segment, then
    pass, row step, bit of the float4, lane), and the per-warp counts"""
    H, W = m.shape
    o = owners(H, W, route)
    keep = peak_mask(m) & (m > floor)
    ys, xs = np.nonzero(keep)
    if route == "scalar":
        nth = np.zeros(len(ys), np.int64)
    else:   # a thread's k-th peak within its float4 goes out in the k-th ballot round
        grp = o["u"][ys, xs] * 1_000_000 + ys
        nth = np.array([int(np.sum((grp == grp[i]) & (xs < xs[i]))) for i in range(len(ys))], np.int64)
    key = [tuple(int(o[k][yy, xx]) for k in ("warp", "pas", "row")) + (int(n), int(o["lane"][yy, xx]))
           for yy, xx, n in zip(ys, xs, nth)]
    order = sorted(range(len(ys)), key=lambda i: key[i])
    vals = m[ys, xs][order]
    idx = (ys * W + xs)[order]
    counts = np.bincount(o["warp"][ys, xs], minlength=TPB // 32)
    return vals.astype(F32), idx.astype(np.int64), counts


def select_rounds(vals, K):
    """select_set's outcome on candidate values ``vals`` (all > 0): ('all', 0) when n <= K, else one of 'take_whole',
    'resolve', 'give_up' with the number of histogram rounds it took, and for 'resolve' the boundary-bucket size"""
    n = len(vals)
    if n <= K:
        return "all", 0, 0
    u = vals.view(np.uint32).astype(np.int64)
    lo, hi, need = int(u.min()), int(u.max()), K
    for rnd in range(5):
        span = hi - lo
        shift = max(0, span.bit_length() - 8) if span else 0
        inr = (u >= lo) & (u <= hi)
        hist = np.bincount((u[inr] - lo) >> shift, minlength=256)
        suf = np.cumsum(hist[::-1])[::-1]
        excl = suf - hist
        tb = int(np.nonzero((excl < need) & (need <= suf))[0][0])
        need_b, nb = need - int(excl[tb]), int(hist[tb])
        if nb == need_b:
            return "take_whole", rnd + 1, nb
        if nb <= BND:
            return "resolve", rnd + 1, nb
        if shift == 0:
            return "give_up", rnd + 1, nb
        need = need_b
        lo = lo + (tb << shift)
        hi = min(hi, lo + (1 << shift) - 1)
    return "give_up", 5, 0


def channel_facts(m, K, is_centre, route):
    """what phase 1 and 2 do with one (H, W) map: dict(n, counts, overflow, select=(outcome, rounds, nb), slow)"""
    floor = F32(0) if is_centre else THRESH
    vals, idx, counts = candidates(m, floor, route)
    overflow = bool(counts.max() > SEG)
    sel = select_rounds(vals, K) if not overflow else ("overflow", 0, 0)
    negative_peak = bool((peak_mask(m) & (m < 0)).any())
    slow = overflow or sel[0] == "give_up" or (is_centre and len(vals) < K and negative_peak)
    return dict(vals=vals, idx=idx, counts=counts, n=len(vals), overflow=overflow, select=sel, slow=slow,
                negative_peak=negative_peak)


def _kth_tied(vals, K):
    s = np.sort(vals)[::-1]
    return len(s) > K and s[K - 1] == s[K]


def seam_facts(m, route):
    """seam branches the peaks of one map reach"""
    H, W = m.shape
    o = owners(H, W, route)
    pk = peak_mask(m) & (m > 0)
    out = set()
    for dy, dx in ((0, 1), (1, 0), (1, 1), (1, -1)):
        ya, yb = slice(0, H - dy), slice(dy, H)
        xa, xb = (slice(0, W - dx), slice(dx, W)) if dx >= 0 else (slice(1, W), slice(0, W - 1))
        a_pk, b_pk = pk[ya, xa], pk[yb, xb]
        either = a_pk | b_pk
        if route != "scalar":
            if dx == 0 and (either & (o["strip"][ya, xa] != o["strip"][yb, xb])).any():
                out.add("seam_strip")
            if dy == 0 and (either & (o["group"][ya, xa] != o["group"][yb, xb])).any():
                out.add("seam_float4")
        if (either & (o["warp"][ya, xa] != o["warp"][yb, xb])).any():
            out.add("seam_warp")
        if (a_pk & b_pk & (m[ya, xa] == m[yb, xb]) & (o["u"][ya, xa] != o["u"][yb, xb])).any():
            out.add("seam_plateau")
    if pk[0, 0] and pk[0, -1] and pk[-1, 0] and pk[-1, -1]:
        out.add("seam_corner")
    return out


def grouping_facts(inp: Inputs, route):
    """grouping branches reached, from the oracle's own quantities (score-sorted candidate list, fp32 squared and
    rounded distances, boxes) plus the kernel's candidate order for the half-CTA split"""
    d = inp.maps
    B, H, W, J = inp.shape
    K = inp.K
    out = set()
    det = decode_ref.multi_pose_decode(d["heat"], d["wh"], d["kps"], d["reg"] if inp.use_reg else None, d["hm_hp"],
                                       d["hp_offset"] if inp.use_off else None, K=K)
    heat = decode_ref.nms3x3(d["heat"])
    _, inds, _, ys, xs = decode_ref.topk(heat, K)
    hm = decode_ref.nms3x3(d["hm_hp"])
    score, hidx, hy, hx = decode_ref.topk_channel(hm, K)
    if inp.use_off:
        off = decode_ref.gather_nchw(d["hp_offset"], hidx.reshape(B, -1)).reshape(B, J, K, 2)
        hx, hy = hx + off[..., 0], hy + off[..., 1]
    else:
        hx, hy = hx + F32(0.5), hy + F32(0.5)
    live = score > THRESH
    kg = decode_ref.gather_nchw(d["kps"], inds).reshape(B, K, J, 2)
    kx = (kg[..., 0] + xs[:, :, None]).transpose(0, 2, 1)            # (B, J, K persons)
    ky = (kg[..., 1] + ys[:, :, None]).transpose(0, 2, 1)
    box = det[:, :, 0:4]
    hk = (K + 1) // 2
    for b in range(B):
        for j in range(J):
            lv = np.nonzero(live[b, j])[0]
            if not len(lv):
                continue
            order = None
            if K % 2 and len(lv) <= K:       # the kernel's list order is deterministic only when no select ran
                _, kidx, _ = candidates(d["hm_hp"][b, j], THRESH, route)
                order = {int(v): i for i, v in enumerate(kidx)}
            for p in range(K):
                dx = (kx[b, j, p] - hx[b, j, lv]).astype(F32)
                dy = (ky[b, j, p] - hy[b, j, lv]).astype(F32)
                sq = (dx * dx).astype(F32) + (dy * dy).astype(F32)
                dist = np.sqrt(sq).astype(F32)
                tied = np.nonzero(dist == dist.min())[0]
                c = lv[tied[0]]                                        # the reference's first minimum
                if len(tied) > 1:
                    if len(set(sq[tied].tolist())) > 1:
                        if sq[tied[0]] > sq[tied].min():
                            out.add("group_sqrt_tie")
                        elif hidx[b, j, c] > hidx[b, j, lv[tied]].min():
                            out.add("group_sqrt_tie_swapped")
                    else:
                        sc = score[b, j, lv[tied]]
                        out.add("group_sq_tie_score" if sc.max() > sc.min() else "group_sq_tie_index")
                    if order is not None:
                        sides = {order[int(hidx[b, j, lv[t]])] < hk for t in tied}
                        if len(sides) == 2:
                            out.add("group_tie_across_halves")
                l, t, r, bt = box[b, p]
                sx, sy, md = hx[b, j, c], hy[b, j, c], dist.min()
                lim = (np.maximum(bt - t, r - l) * F32(0.3)).astype(F32)
                kept = not (sx < l or sx > r or sy < t or sy > bt or md > lim)
                if kept and (sx == l or sx == r or sy == t or sy == bt):
                    out.add("group_box_edge")
                if kept and md == lim:
                    out.add("group_min_dist_edge")
    return out


def reached(case: DecodeCase, inp: Inputs = None):
    """every branch of ``BRANCHES`` the case's data reaches, computed from the maps"""
    inp = inp or case.build()
    d = inp.maps
    B, H, W, J = inp.shape
    K = inp.K
    route = scan_route(H, W, not inp.misaligned)
    out = set()
    if route == "w128":
        out.add("scan_w128")
    elif route == "vec":
        out.add("scan_vec")
        if (W // 4) % 32:
            out.add("scan_vec_shared_warp")
        if W // 4 > TPB:
            out.add("scan_vec_two_pass")
    else:
        out.add("scan_scalar_misaligned" if W % 4 == 0 else "scan_scalar")
    seams = None
    for b in range(B):
        for ch in range(1 + J):
            m = d["heat"][b, 0] if ch == 0 else d["hm_hp"][b, ch - 1]
            s = seam_facts(m, route)
            seams = s if seams is None else seams & s          # a seam counts when every map of the case has it
            f = channel_facts(m, K, ch == 0, route)
            who = "centre" if ch == 0 else "joint"
            if f["overflow"] and f["counts"].sum() <= CAP:
                out.add("segment_overflow")
            outcome, rounds, nb = f["select"]
            if ch == 0 and f["n"] == K:
                out.add("count_eq_k")
            if ch == 0 and f["n"] == K + 1:
                out.add("count_k_plus_1")
            if outcome == "take_whole" and rounds == 1:
                out.add(f"{who}:bucket_take_whole")
            if outcome == "resolve" and rounds == 1 and nb >= 2 and _kth_tied(f["vals"], K):
                out.add(f"{who}:bucket_resolve_ties")
            if outcome in ("take_whole", "resolve") and rounds >= 2:
                out.add(f"{who}:bucket_refine")
            if outcome in ("take_whole", "resolve") and rounds >= 4 and ch == 0:
                out.add("centre:bucket_max_rounds")
            if outcome == "give_up":
                out.add(f"{who}:bucket_give_up")
            if ch == 0 and f["n"] < K:
                if f["negative_peak"]:
                    out.add("fill_negative_peak")
                else:
                    out.add("fill_n_ge_2k" if H * W >= 2 * K else "fill_n_lt_2k")
                    if not m.any():
                        out.add("fill_all_zero")
                    if (np.signbit(m) & (m == 0)).any():
                        out.add("fill_neg_zero")
            if ch > 0:
                if f["n"] == 0:
                    out.add("mask_no_candidate")
                if f["n"] > K and _kth_tied(f["vals"], K):
                    out.add("mask_over_k_ties")
                pk = peak_mask(m)
                if (pk & (m == THRESH)).any() and (pk & (m == np.nextafter(THRESH, F32(1)))).any():
                    out.add("mask_exact_thresh")
    out |= seams or set()
    out |= grouping_facts(inp, route)
    if K == 1:
        out.add("group_k1")
    if not inp.use_reg and not inp.use_off:
        out.add("group_no_reg_off")
    if B >= 48 and J == 17 and len({d["heat"][b].tobytes() for b in range(B)}) == B:
        out.add("batch_many_ctas")
    if J == 1:
        out.add("joints_1")
    if J == MAXJ:
        out.add("joints_32")
    return out


# ------------------------------------------------------------------------------------------------------ builders
def _base(B, H, W, J=17, seed=0, kind="smooth"):
    """a synth_decode_inputs base (random regressions) with the heat maps cleared"""
    d = decode_ref.synth_decode_inputs(B, H, W, seed=seed, J=J, kind=kind)
    d["heat"][:] = 0
    d["hm_hp"][:] = 0
    return d


def _seam_map(H, W, route, rng, top):
    """a uniform [0, 0.25) background with peaks placed on every seam the route has: the four corners, then pairs of
    neighbouring cells owned by different strips, float4 groups or warps.  Each pair gets a peak on one side and the
    next float below it on the other (so the lower cell is a non-peak only through its neighbour across the seam), in
    both directions, or an equal plateau.  Peak values start at ``top`` and fall by 2^-10 (all exact)."""
    m = rng.uniform(0, 0.25, size=(H, W)).astype(F32)
    o = owners(H, W, route)
    used = np.zeros((H, W), bool)
    val = [top]

    def nxt():
        v = F32(val[0])
        val[0] = F32(val[0] - F32(2 ** -10))
        return v

    def free(cells):
        for (y, x) in cells:
            if used[max(0, y - 1):y + 2, max(0, x - 1):x + 2].any():
                return False
        return True

    def mark(cells):
        for (y, x) in cells:
            used[y, x] = True

    for (y, x) in ((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)):
        if free([(y, x)]):
            v = nxt(); m[y, x] = v; mark([(y, x)])
    pairs = {"strip": [], "group": [], "warp": []}
    for y in range(H):
        for x in range(W):
            for dy, dx in ((0, 1), (1, 0)):
                yy, xx = y + dy, x + dx
                if yy >= H or xx >= W:
                    continue
                for k in pairs:
                    if o[k][y, x] != o[k][yy, xx] and (k != "strip" or o["strip"][y, x] >= 0) and \
                            (k != "group" or o["group"][y, x] >= 0):
                        pairs[k].append(((y, x), (yy, xx)))
    for k, lst in pairs.items():
        if not lst:
            continue
        pick = [lst[i] for i in np.linspace(0, len(lst) - 1, num=min(len(lst), 12)).astype(int)]
        for i, (a, b) in enumerate(pick):
            if not free([a, b]):
                continue
            v = nxt()
            if i % 3 == 2:
                m[a], m[b] = v, v                                   # plateau across the seam: both kept
            else:
                hi_, lo_ = (a, b) if i % 3 == 0 else (b, a)
                m[hi_], m[lo_] = v, np.nextafter(v, F32(0))
            mark([a, b])
    return m


def scan_case(name, B, H, W, misaligned, K, reason, branches, J=17, seed=0):
    route = scan_route(H, W, not misaligned)

    def build():
        rng = np.random.RandomState(seed)
        d = _base(B, H, W, J, seed)
        for b in range(B):
            d["heat"][b, 0] = _seam_map(H, W, route, rng, F32(0.9))
            for j in range(J):
                d["hm_hp"][b, j] = _seam_map(H, W, route, rng, F32(0.9))
        return Inputs(d, K, misaligned=misaligned)
    seams = {"seam_corner", "seam_warp", "seam_plateau"}
    if route != "scalar":
        seams |= {"seam_float4"} | ({"seam_strip"} if owners(H, W, route)["strip"].max() > 0 else set())
    add(name, build, reason, *branches, *seams)


scan_case("scan_w128_64x128", 1, 64, 128, False, 100, "scan_w128: peaks on the 8-row strip seams (warp seams too), "
          "float4 seams, corners; plateaus across them", ["scan_w128"], J=3)
scan_case("scan_vec_12x128", 1, 12, 128, False, 100, "scan_vec at W = 128 with H % 8 != 0: 2-row strips, the last "
          "two warps without rows", ["scan_vec"], J=3)
scan_case("scan_vec_40x40", 2, 40, 40, False, 100, "scan_vec with XG = 10: 25 strips of 2 rows, a warp spans 3.2 "
          "strips, lane 31 | lane 0 falls inside a strip's row", ["scan_vec", "scan_vec_shared_warp"], J=3)
scan_case("scan_vec_8x1100", 1, 8, 1100, False, 100, "scan_vec with XG = 275 > 256: one strip, two passes, the "
          "second pass's lane 0 reads its left neighbour from memory", ["scan_vec", "scan_vec_two_pass"], J=2)
scan_case("scan_scalar_30x37", 1, 30, 37, False, 100, "scan_scalar: W = 37, warp seams inside rows and at the "
          "256-cell pass boundary", ["scan_scalar"], J=3)
scan_case("scan_scalar_misaligned_32x64", 1, 32, 64, True, 100, "W = 64 from a view one float past a 16-byte "
          "boundary: vec_ok fails on alignment alone", ["scan_scalar_misaligned"], J=3)


def _isolated_slots(H, W, rng):
    """cells 2 apart in both directions (each its own 3x3 neighbourhood), shuffled"""
    ys, xs = np.mgrid[0:H:2, 0:W:2]
    cells = np.stack([ys.ravel(), xs.ravel()], 1)
    return cells[rng.permutation(len(cells))]


def _place(m, vals, slots):
    assert len(vals) <= len(slots)
    for v, (y, x) in zip(vals, slots):
        m[y, x] = v


def _spread(n, lo, hi):
    """n distinct exact fp32 values evenly spread over [lo, hi]"""
    v = np.linspace(lo, hi, n).astype(F32)
    assert len(np.unique(v)) == n
    return v


def _ulps(v, n, dup=0):
    """n consecutive floats from v upwards, the first ``dup`` of them twice"""
    out = [F32(v)]
    for _ in range(n - 1):
        out.append(np.nextafter(out[-1], F32(2)))
    return np.array(out + out[:dup], F32)


def count_case(name, n_centre, K, branches, reason):
    def build():
        rng = np.random.RandomState(len(name))
        d = _base(1, 64, 64, 17, seed=len(name))
        _place(d["heat"][0, 0], _spread(n_centre, 0.2, 0.9), _isolated_slots(64, 64, rng))
        _place(d["hm_hp"][0, 0], _spread(K, 0.2, 0.9), _isolated_slots(64, 64, rng))
        _place(d["hm_hp"][0, 1], _spread(K + 1, 0.2, 0.9), _isolated_slots(64, 64, rng))
        return Inputs(d, K)
    add(name, build, reason, *branches)


count_case("count_eq_k", 50, 50, ["count_eq_k"], "exactly K candidates in the centre map and in joint 0: select_set "
           "copies them all (n <= K)")
count_case("count_k_plus_1", 51, 50, ["count_k_plus_1"], "K + 1 candidates: the smallest bucket select, one key "
           "left out")


def _overflow():
    """rows 0..15 of a 128x128 map (warp 0's strip in scan_w128): equal horizontal pairs at columns 3i, 3i+1 on every
    even row = 43 pairs x 2 x 8 rows = 688 candidates in one segment; the rest of the map is a sparse sprinkle"""
    rng = np.random.RandomState(41)
    d = _base(1, 128, 128, 17, seed=41)
    for m in (d["heat"][0, 0], d["hm_hp"][0, 4]):
        v = 0.2
        for y in range(0, 16, 2):
            for x in range(0, 128, 3):
                m[y, x:x + 2] = F32(v)
                v += 2 ** -12
        slots = [s for s in _isolated_slots(128, 128, rng) if s[0] >= 18]
        _place(m, _spread(300, 0.3, 0.95), slots)
    d["hm_hp"][0, :4] = d["heat"][0, 0]
    return Inputs(d, 100)


add("segment_overflow", _overflow, "one warp's strip holds 688 candidates (> 512) while the map holds under 4096: "
    "compact_segments overflows into select_slow, which must still find equal-pair plateaus in index order",
    "segment_overflow")


def bucket_case(name, K, cluster, need_in_cluster, branches, reason, span=None):
    """a high group (K - need_in_cluster distinct values in [0.7, 0.95]), the ``cluster`` values at the K-th rank and
    200 distinct low values, in the centre map and in joint 2 (whose floor is 0.1); ``span`` adds the extreme values of
    the centre map"""
    def build():
        rng = np.random.RandomState(7 + len(name))
        d = _base(1, 64, 64, 17, seed=7)
        high = _spread(K - need_in_cluster, 0.7, 0.95)
        low = _spread(200, 0.15, 0.3)
        vals = np.concatenate([high, cluster, low])
        _place(d["hm_hp"][0, 2], vals, _isolated_slots(64, 64, rng))
        if span is not None:
            vals = np.concatenate([vals, np.array(span, F32)])
        _place(d["heat"][0, 0], vals, _isolated_slots(64, 64, rng))
        return Inputs(d, K)
    add(name, build, reason, *branches)


bucket_case("bucket_take_whole", 100, np.full(10, F32(0.5)), 10, ["centre:bucket_take_whole", "joint:bucket_take_whole"],
            "10 exact ties form the boundary bucket and all 10 are needed: taken whole, no rank counting")
bucket_case("bucket_resolve_ties", 100, np.full(20, F32(0.5)), 10,
            ["centre:bucket_resolve_ties", "joint:bucket_resolve_ties", "mask_over_k_ties"],
            "20 exact ties at the K-th value, 10 needed: rank counting on (value, ~index) keeps the 10 lowest indices")
bucket_case("bucket_refine", 100, _ulps(0.5, 100), 50, ["centre:bucket_refine", "joint:bucket_refine"],
            "100 distinct values within 100 ulps at the K-th rank: the first boundary bucket holds > 64, one refine "
            "round separates them")
bucket_case("bucket_give_up", 100, np.full(100, F32(0.5)), 50, ["centre:bucket_give_up", "joint:bucket_give_up"],
            "100 exact ties at the K-th value: > 64 ties at shift 0, select_set gives up to select_slow")
def _max_rounds_cluster():
    """62 consecutive floats (8 of them twice) from the first start at or above 0.5 whose cluster falls inside one
    64-float bucket of the third round, so that a fourth round (shift 0) is needed"""
    high, low = _spread(65, 0.7, 0.95), _spread(200, 0.15, 0.3)
    v = F32(0.5)
    for _ in range(64):
        c = _ulps(v, 62, dup=8)
        if select_rounds(np.concatenate([high, c, low, np.array([1e-38, 1.0], F32)]), 100)[1] >= 4:
            return c
        v = np.nextafter(v, F32(1))
    raise AssertionError("no start puts the cluster in one third-round bucket")


bucket_case("bucket_max_rounds", 100, _max_rounds_cluster(), 35, ["centre:bucket_max_rounds", "centre:bucket_refine"],
            "a centre value span from 1e-38 (subnormal) to 1.0: histogram shifts 22, 14, 6, 0 before the 70-key "
            "cluster (8 duplicated) is resolved", span=[1e-38, 1.0])


def fill_case(name, H, W, K, branches, reason, edit):
    def build():
        d = _base(1, H, W, 17, seed=H * W + K)
        edit(d, np.random.RandomState(H + W))
        return Inputs(d, K)
    add(name, build, reason, *branches)


def _few(n):
    def edit(d, rng):
        H, W = d["heat"].shape[2:]
        _place(d["heat"][0, 0], _spread(n, 0.2, 0.9), _isolated_slots(H, W, rng))
        for j in range(3):
            _place(d["hm_hp"][0, j], _spread(n, 0.2, 0.9), _isolated_slots(H, W, rng))
    return edit


def _neg_zero(d, rng):
    _few(5)(d, rng)
    H, W = d["heat"].shape[2:]
    z = (rng.uniform(size=(H, W)) < 0.3) & (d["heat"][0, 0] == 0)
    d["heat"][0, 0][z] = F32(-0.0)


def _neg_peak(d, rng):
    H, W = d["heat"].shape[2:]
    d["heat"][0, 0] = F32(-0.5)
    d["heat"][0, 0, 6, 6] = F32(-0.25)                           # a negative 3x3 maximum
    _place(d["heat"][0, 0], _spread(4, 0.2, 0.9), [(0, 0), (2, 9), (10, 3), (11, 11)])


fill_case("fill_few_32x32", 32, 32, 100, ["fill_n_ge_2k"], "30 positive peaks, K = 100, H*W >= 2K: the 70 zero rows "
          "are the lowest free flat indices", _few(30))
fill_case("fill_few_9x13", 9, 13, 100, ["fill_n_lt_2k"], "6 positive peaks, K = 100 on 117 cells: the free cells run "
          "out of the first 2K before they run out of the map", _few(6))
fill_case("fill_all_zero", 16, 16, 50, ["fill_all_zero", "fill_n_ge_2k"], "no centre candidate at all",
          lambda d, rng: None)
fill_case("fill_neg_zero", 20, 20, 60, ["fill_neg_zero", "fill_n_ge_2k"], "-0.0 cells equal 0 for the NMS and the "
          "ordering; the fill must not take them for negative peaks", _neg_zero)
fill_case("fill_negative_peak", 12, 12, 100, ["fill_negative_peak"], "a negative peak beside four positive ones: the "
          "zero cells no longer rank last, select_slow decides", _neg_peak)


def _kind(kind, K, J=17):
    return lambda: Inputs(decode_ref.synth_decode_inputs(1, 40, 40, seed=0, J=J, kind=kind), K)


add("thresh", _kind("thresh", 10), "keypoint peaks of exactly fp32(0.1) two cells from each guess are masked; the "
    "nextafter(0.1, 1) ones four rows away are kept and chosen; joint 16 has only the masked ones",
    "mask_exact_thresh", "mask_no_candidate")
add("sqrttie", _kind("sqrttie", 10), "equal fp32 sqrt, squared distances one ulp apart: the reference takes B, the "
    "first in score order, though A's squared distance is smaller", "group_sqrt_tie")
add("sqrttie_swap", _kind("sqrttie_swap", 10), "the same with the scores swapped: A is first in score order with the "
    "higher flat index", "group_sqrt_tie_swapped")
add("sqtie", _kind("sqtie", 10), "exactly equal squared distances: the higher score wins (joint 0 at the higher flat "
    "index, joint 1 at the lower)", "group_sq_tie_score")


def _sqtie_equal():
    inp = _kind("sqtie", 10)()
    inp.maps["hm_hp"][:, 0][inp.maps["hm_hp"][:, 0] > 0] = F32(0.55)
    return inp


add("sqtie_equal_scores", _sqtie_equal, "exactly equal squared distances and equal scores: the lower flat index wins",
    "group_sq_tie_index")


def _halves():
    """41x41 (scan_scalar), K = 5, hk = 3.  One person at cell (20,20) with guess (20.0, 20.5); candidates at cells
    (22,20) (flat 922, warp 4: list position 0) and (18,20) (flat 758, warp 7: position 3) land at (20.0, 22.5) and
    (20.0, 18.5), dy = -+2 exactly; two far fillers in warps 5 and 6 take positions 1 and 2.  Joint 0: equal scores
    (the lower index, in the second half, wins); joint 1: the higher score in the second half; joint 2: in the first."""
    d = _base(1, 41, 41, 17, seed=3)
    heat, hm, off, kps = d["heat"][0, 0], d["hm_hp"][0], d["hp_offset"][0], d["kps"][0]
    heat[20, 20] = F32(0.9)
    d["wh"][0, :, 20, 20] = F32(30)
    for j, (s_hi, s_lo) in enumerate(((0.5, 0.5), (0.5, 0.6), (0.6, 0.5))):
        kps[2 * j:2 * j + 2, 20, 20] = (F32(0), F32(0.5))
        hm[j, 22, 20] = F32(s_hi); hm[j, 18, 20] = F32(s_lo)
        for cell in (180, 215):                                    # warps 5 and 6 of iteration 0
            hm[j, cell // 41, cell % 41] = F32(0.3)
    off[:, 22, 20] = (F32(0), F32(0.5))
    off[:, 18, 20] = (F32(0), F32(0.5))
    return Inputs(d, 5)


add("tie_across_halves", _halves, "K = 5: the tied pair sits at list positions 0 and 3, one in each half-CTA range "
    "(hk = 3); the merge of the halves must apply the same tie rule", "group_tie_across_halves", "group_sq_tie_index",
    "group_sq_tie_score")


def _edges():
    """person at cell (20,20), reg (0.5, 0.5), wh (10, 10): box [15.5, 25.5] in x and y, 0.3 * max(h, w) = 3.  Joints
    0..3 have a candidate exactly on l, r, t, b; joint 4 one float left of l (rejected); joint 5 a candidate at
    exactly the distance limit (kept), joint 6 one float past it (rejected)."""
    d = _base(1, 40, 40, 17, seed=5)
    heat, hm, off, kps = d["heat"][0, 0], d["hm_hp"][0], d["hp_offset"][0], d["kps"][0]
    heat[20, 20] = F32(0.9)
    d["wh"][0, :, 20, 20] = F32(10)
    d["reg"][0, :, 20, 20] = F32(0.5)
    lim = F32(F32(10) * F32(0.3))
    put = [  # joint, kps offset (guess = cell + offset), candidate cell, hp_offset
        (0, (-3.0, 0.5), (20, 15), (0.5, 0.5)),
        (1, (3.0, 0.5), (20, 25), (0.5, 0.5)),
        (2, (0.5, -3.0), (15, 20), (0.5, 0.5)),
        (3, (0.5, 3.0), (25, 20), (0.5, 0.5)),
        (4, (-3.0, 0.5), (21, 15), (float(np.nextafter(F32(15.5), F32(0)) - F32(15)), -0.5)),
        (5, (0.0, 0.5), (20, 23), (float(lim - F32(3)), 0.5)),
        (6, (0.0, 0.5), (19, 23), (float(np.nextafter(F32(23), F32(99)) - F32(23)), 1.5)),
    ]
    for j, kp, (cy, cx), (ox, oy) in put:
        kps[2 * j:2 * j + 2, 20, 20] = (F32(kp[0]), F32(kp[1]))
        hm[j, cy, cx] = F32(0.5)
        off[:, cy, cx] = (F32(ox), F32(oy))
    return Inputs(d, 10)


add("box_and_distance_edges", _edges, "candidates exactly on each box edge and at exactly 0.3 * max(h, w) are kept "
    "(the tests are < , > and >); one float further they are rejected", "group_box_edge", "group_min_dist_edge")


def _smooth(B, H, W, K, J=17, seed=0, use_reg=True, use_off=True):
    return lambda: Inputs(decode_ref.synth_decode_inputs(B, H, W, seed=seed, J=J, kind="smooth"), K, use_reg, use_off)


add("k1", _smooth(2, 64, 64, 1, seed=61), "K = 1: one person per image, hk = 1, the second half-CTA scans nothing",
    "group_k1")
add("no_reg_no_offset", _smooth(2, 64, 64, 50, seed=62, use_reg=False, use_off=False), "reg and hp_offset None: "
    "centres and keypoint candidates at cell + 0.5", "group_no_reg_off")
add("joints_1", _smooth(2, 48, 64, 60, J=1, seed=63), "J = 1: two CTAs per image, the last joint is the first",
    "joints_1")
add("joints_32", _smooth(2, 48, 64, 60, J=32, seed=64), "J = 32 = CPB200_DECODE_MAX_J: 33 CTAs per image, 101-float "
    "rows", "joints_32")
add("batch_48", _smooth(48, 64, 64, 100, seed=65), "B = 48, J = 17: 864 CTAs, more than are resident at once; every "
    "joint CTA waits on its own image's centre CTA", "batch_many_ctas")

CASE = {c.name: c for c in CASES}
assert len(CASE) == len(CASES)
