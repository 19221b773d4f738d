"""GPU parity tests of the fused decode kernel (through the C ABI) against the oracle and the
reference-generated golden vectors.  Integer/index work is bit-exact; float columns are
produced with the reference's operation order and compared with tolerance 1e-5 (written
here; the north-star bound is 1e-3)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import decode_ref

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-5
DEV = "cuda:0"


def _cuda_decode(inp, K, use_reg=True, use_off=True, apply_sigmoid=False):
    from centerpose_b200 import multi_pose_decode
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in inp.items()}
    out = multi_pose_decode(t["heat"], t["wh"], t["kps"], reg=t["reg"] if use_reg else None,
                            hm_hp=t["hm_hp"], hp_offset=t["hp_offset"] if use_off else None, K=K,
                            apply_sigmoid=apply_sigmoid)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _oracle(inp, K, use_reg=True, use_off=True):
    return decode_ref.multi_pose_decode(inp["heat"], inp["wh"], inp["kps"], inp["reg"] if use_reg else None,
                                        inp["hm_hp"], inp["hp_offset"] if use_off else None, K=K)


def _assert_same(got, ref, only_positive=False):
    assert got.shape == ref.shape
    if only_positive:
        m = ref[:, :, 4] > 0
        got, ref = got[m], ref[m]
    bad = np.abs(got - ref) > TOL * np.maximum(1.0, np.abs(ref))
    assert not bad.any(), f"{int(bad.sum())} elements differ, max {np.abs(got - ref).max()}"


DECODE_FILES = sorted(glob.glob(os.path.join(GOLD, "decode_*.npz")))


@pytest.mark.parametrize("path", DECODE_FILES, ids=[os.path.basename(p)[7:-4] for p in DECODE_FILES])
def test_decode_matches_reference_golden(path):
    g = np.load(path)
    B, H, W, K, seed, use_reg, use_off = [int(v) for v in g["meta"]]
    inp = decode_ref.synth_decode_inputs(B, H, W, seed=seed, kind=str(g["kind"]))
    got = _cuda_decode(inp, K, bool(use_reg), bool(use_off))
    _assert_same(got, g["det"], only_positive=True)          # vs the reference's own output
    _assert_same(got, _oracle(inp, K, bool(use_reg), bool(use_off)))   # vs the oracle, every row


@pytest.mark.parametrize("kind,B,H,W,K", [
    ("smooth", 3, 128, 128, 100), ("uniform", 2, 128, 128, 100), ("uniform", 1, 256, 256, 100),
    ("plateau", 1, 32, 32, 20), ("sparse", 2, 128, 128, 100), ("lowhp", 2, 64, 64, 100),
    ("smooth", 2, 30, 37, 50), ("uniform", 1, 9, 13, 100), ("smooth", 1, 128, 128, 1),
    ("smooth", 1, 128, 128, 128), ("uniform", 2, 96, 200, 77), ("smooth", 1, 8, 1100, 64),
])
def test_decode_matches_oracle(kind, B, H, W, K):
    inp = decode_ref.synth_decode_inputs(B, H, W, seed=1000 + H + W + K, kind=kind)
    _assert_same(_cuda_decode(inp, K), _oracle(inp, K))


def test_decode_single_joint_and_misaligned_views():
    inp = decode_ref.synth_decode_inputs(2, 40, 44, seed=4, J=1)
    _assert_same(_cuda_decode(inp, 30), _oracle(inp, 30))
    from centerpose_b200 import multi_pose_decode
    big = decode_ref.synth_decode_inputs(1, 33, 44, seed=5)
    t = {k: torch.from_numpy(v).cuda() for k, v in big.items()}
    sl = {k: v[:, :, 1:, :] for k, v in t.items()}      # non-contiguous -> shim makes it contiguous
    out = multi_pose_decode(sl["heat"], sl["wh"], sl["kps"], sl["reg"], sl["hm_hp"], sl["hp_offset"], K=40)
    ref = _oracle({k: np.ascontiguousarray(v[:, :, 1:, :]) for k, v in big.items()}, 40)
    _assert_same(out.cpu().numpy(), ref)


def test_decode_negative_map_takes_exact_path():
    inp = decode_ref.synth_decode_inputs(1, 12, 12, seed=9, kind="uniform")
    inp["heat"] = (inp["heat"] - 2.0).astype(np.float32)      # all-negative centre map
    _assert_same(_cuda_decode(inp, 100), _oracle(inp, 100))


def test_decode_fused_sigmoid():
    """apply_sigmoid=True on logits == decode(sigmoid(logits)); scores within 1e-6, rows matched
    tie-insensitively (the fused logistic uses ex2.approx; order of near-equal scores may flip)."""
    from tests.util import match_rows
    inp = decode_ref.synth_decode_inputs(2, 128, 128, seed=21, kind="smooth")
    logit = lambda p: np.log(p / (1 - p)).astype(np.float32)
    lin = dict(inp); lin["heat"] = logit(np.clip(inp["heat"], 1e-6, 1 - 1e-6)); lin["hm_hp"] = logit(np.clip(inp["hm_hp"], 1e-6, 1 - 1e-6))
    sig = lambda a: torch.from_numpy(a).sigmoid().numpy()
    ref = _oracle(dict(inp, heat=sig(lin["heat"]), hm_hp=sig(lin["hm_hp"])), 100)
    got = _cuda_decode(lin, 100, apply_sigmoid=True)
    for b in range(2):
        rows, elems = match_rows(got[b], ref[b], tol=1e-4)
        assert rows >= 0.97 and elems >= 0.97, (rows, elems)


def test_decode_full_size_properties():
    """BASELINE config-2 size (B=32, 128x128): size-independent properties."""
    from centerpose_b200 import multi_pose_decode
    B, H, W, K = 32, 128, 128, 100
    inp = decode_ref.synth_decode_inputs(B, H, W, seed=77, kind="smooth")
    t = {k: torch.from_numpy(v).cuda() for k, v in inp.items()}
    run = lambda: multi_pose_decode(t["heat"], t["wh"], t["kps"], t["reg"], t["hm_hp"], t["hp_offset"], K=K)
    a = run(); b = run(); torch.cuda.synchronize()
    assert torch.equal(a, b)                                   # deterministic, workspace self-cleans
    sc = a[:, :, 4]
    assert bool((sc[:, :-1] >= sc[:, 1:]).all())              # sorted descending
    # every reported centre is a 3x3 local maximum whose value is the reported score
    heat = t["heat"]; hmax = torch.nn.functional.max_pool2d(heat, 3, 1, 1)
    peaks = (heat * (hmax == heat).float()).view(B, -1)
    kth = peaks.topk(K, dim=1).values
    assert torch.equal(kth, sc)                                # exact top-K multiset (values)
    cx = (a[:, :, 0] + a[:, :, 2]) * 0.5; cy = (a[:, :, 1] + a[:, :, 3]) * 0.5
    assert bool((cx > -1).all() and (cx < W + 1).all() and (cy > -1).all() and (cy < H + 1).all())
    # oracle on a slice of the batch
    ref = _oracle({k: v[:4] for k, v in inp.items()}, K)
    _assert_same(a[:4].cpu().numpy(), ref)


def test_decode_fused_post_process():
    """decode + fused back-projection == oracle decode followed by the oracle's multi_pose_post_process
    (which is pinned against the reference).  Tolerance 2e-3 px on coordinates up to ~2000 px (fp32 affine on the
    device vs the reference's float64)."""
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.decode import affine_for_meta
    from oracle import post_process_ref
    B, H, W, K = 3, 128, 128, 100
    inp = decode_ref.synth_decode_inputs(B, H, W, seed=55, kind="smooth")
    metas = [post_process_ref.make_meta(480, 640, 1.0, True), post_process_ref.make_meta(1080, 1920, 1.0, True),
             post_process_ref.make_meta(333, 500, 1.0, True)]
    t = {k: torch.from_numpy(v).cuda() for k, v in inp.items()}
    got = multi_pose_decode(t["heat"], t["wh"], t["kps"], t["reg"], t["hm_hp"], t["hp_offset"], K=K,
                            affine=affine_for_meta(metas).cuda()).cpu().numpy()
    ref = _oracle(inp, K)
    for b in range(B):
        want = post_process_ref.multi_pose_post_process(ref[b:b + 1].copy(), [metas[b]["c"]], [metas[b]["s"]],
                                                        metas[b]["out_height"], metas[b]["out_width"])[0][1]
        assert np.abs(got[b] - want).max() <= 2e-3, np.abs(got[b] - want).max()


def test_decode_error_behaviour():
    from centerpose_b200 import multi_pose_decode
    inp = decode_ref.synth_decode_inputs(1, 8, 8, seed=2)
    t = {k: torch.from_numpy(v).cuda() for k, v in inp.items()}
    with pytest.raises(RuntimeError):      # torch.topk: "selected index k out of range"
        multi_pose_decode(t["heat"], t["wh"], t["kps"], t["reg"], t["hm_hp"], t["hp_offset"], K=100)
    with pytest.raises(NameError):         # decode.py:307 in the reference
        multi_pose_decode(t["heat"], t["wh"], t["kps"], t["reg"], None, None, K=10)
    with pytest.raises(RuntimeError):      # C ABI limit, reported through cpb200_last_error
        big = decode_ref.synth_decode_inputs(1, 32, 32, seed=2)
        tb = {k: torch.from_numpy(v).cuda() for k, v in big.items()}
        multi_pose_decode(tb["heat"], tb["wh"], tb["kps"], tb["reg"], tb["hm_hp"], tb["hp_offset"], K=129)
    with pytest.raises(RuntimeError):      # CPU tensors are rejected (like _ext, dcn_v2.h:38)
        multi_pose_decode(*[torch.from_numpy(inp[k]) for k in ("heat", "wh", "kps")])


def test_flip_merge_matches_reference_helpers():
    """cpb200_flip_merge vs the reference's flip_tensor / flip_lr / flip_lr_off (golden, lib/models/utils.py:27-47)
    and vs the averaging expression of multi_pose.py:45-53 — bit-exact (same fp32 operations)."""
    from centerpose_b200.decode import flip_merge
    g = np.load(os.path.join(GOLD, "flip.npz"))
    idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    hm_hp_f = torch.from_numpy(g["hm_hp"]); hps_f = torch.from_numpy(g["hps"])          # the "mirrored image" maps
    H, W = hm_hp_f.shape[2:]
    gen = torch.Generator().manual_seed(2)
    hm_hp0 = torch.rand(1, 17, H, W, generator=gen); hps0 = torch.randn(1, 34, H, W, generator=gen)
    hm = torch.rand(2, 1, H, W, generator=gen); wh = torch.rand(2, 2, H, W, generator=gen) * 30
    o_hm, o_wh, o_hps, o_hp = flip_merge(hm.to(DEV), wh.to(DEV), torch.cat([hps0, hps_f]).to(DEV),
                                         torch.cat([hm_hp0, hm_hp_f]).to(DEV), idx)
    assert torch.equal(o_hm.cpu(), (hm[0:1] + torch.flip(hm[1:2], [3])) / 2)
    assert torch.equal(o_wh.cpu(), (wh[0:1] + torch.flip(wh[1:2], [3])) / 2)
    assert torch.equal(o_hps.cpu(), (hps0 + torch.from_numpy(g["flip_lr_off"])) / 2)
    assert torch.equal(o_hp.cpu(), (hm_hp0 + torch.from_numpy(g["flip_lr"])) / 2)
    # several pairs, no hm_hp
    hm = torch.rand(6, 1, H, W, generator=gen); wh = torch.rand(6, 2, H, W, generator=gen); hps = torch.randn(6, 34, H, W, generator=gen)
    o_hm, o_wh, o_hps, o_hp = flip_merge(hm.to(DEV), wh.to(DEV), hps.to(DEV), None, idx)
    assert o_hp is None and o_hm.shape[0] == 3
    assert torch.equal(o_hm.cpu(), (hm[0::2] + torch.flip(hm[1::2], [3])) / 2)


def test_soft_nms_cuda_matches_compiled_reference_golden():
    """cpb200_soft_nms_39 on a device array vs golden vectors from the reference's own Cython module
    (oracle/build_ref.py): same keep counts and row movements; scores within 1 float ulp (see the host test)."""
    from centerpose_b200.soft_nms import soft_nms_39, soft_nms_39_cuda
    g = np.load(os.path.join(GOLD, "soft_nms.npz"))
    for boxes, out, keep, prm in zip(g["boxes"], g["out"], g["keep"], g["params"]):
        N, method, Nt, thr = int(prm[0]), int(prm[1]), float(prm[2]), float(prm[3])
        dev = torch.from_numpy(boxes[:N].copy()).to(DEV)
        k = soft_nms_39_cuda(dev, sigma=0.5, Nt=Nt, threshold=thr, method=method)
        assert k == int(keep)
        assert np.abs(dev.cpu().numpy() - out[:N]).max() <= 2e-7
        host = boxes[:N].copy()
        soft_nms_39(host, sigma=0.5, Nt=Nt, threshold=thr, method=method)
        assert np.array_equal(dev.cpu().numpy(), host) or np.abs(dev.cpu().numpy() - host).max() <= 6e-8
    # larger than one pass of the block (N > 128) and the empty case
    rng = np.random.RandomState(5)
    N = 300
    c = rng.uniform(0, 400, size=(N, 2)); wh = rng.uniform(5, 120, size=(N, 2))
    rows = np.zeros((N, 56), np.float32); rows[:, 0:2] = c - wh / 2; rows[:, 2:4] = c + wh / 2
    rows[:, 4] = rng.uniform(0, 1, N); rows[:, 5:] = rng.uniform(0, 400, size=(N, 51))
    host = rows.copy(); kh = len(soft_nms_39(host, Nt=0.5, method=2))
    dev = torch.from_numpy(rows.copy()).to(DEV); kd = soft_nms_39_cuda(dev, Nt=0.5, method=2)
    assert kd == kh and np.abs(dev.cpu().numpy() - host).max() <= 2e-7
    assert soft_nms_39_cuda(torch.zeros(0, 56, device=DEV), Nt=0.5, method=2) == 0


def _bench_maps(B):
    """bench.py's synthetic head maps of its large-batch decode timings, drawn as it draws them: one seed-317 device
    generator for B = 256, then B = 1024."""
    dev = torch.device(DEV)
    g = torch.Generator(device=dev).manual_seed(317)
    for Bd in (256, 1024):
        maps = (torch.randn(Bd, 1, 128, 128, device=dev, generator=g) * 2 - 2.19,
                torch.rand(Bd, 2, 128, 128, device=dev, generator=g) * 40,
                torch.randn(Bd, 34, 128, 128, device=dev, generator=g) * 10,
                torch.rand(Bd, 2, 128, 128, device=dev, generator=g),
                torch.randn(Bd, 17, 128, 128, device=dev, generator=g) * 2 - 2.19,
                torch.rand(Bd, 2, 128, 128, device=dev, generator=g))
        if Bd == B:
            return maps
        del maps


@pytest.mark.parametrize("B", [256, 1024])
def test_decode_at_bench_batches(B):
    """bench.py's decode call (apply_sigmoid=True, K = 100) at B = 256 and 1024, B * 18 CTAs grouping keypoints through
    one release/acquire flag per (image, joint): every image's rows equal a B = 1 call on that image, bit for bit.  On
    maps torch turned into sigmoids (apply_sigmoid=False: the fused logistic uses ex2.approx), slots 0, 1, B // 2, B - 1
    and every multiple of 128 equal the oracle's rows bit for bit.  After every call the workspace's pair counters are
    back at zero."""
    from centerpose_b200 import multi_pose_decode
    from centerpose_b200.decode import _workspace
    K, J = 100, 17
    hm, wh, hps, reg, hm_hp, hpo = _bench_maps(B)

    def decode(b0, b1, heat, joints, sig):
        out = multi_pose_decode(heat[b0:b1], wh[b0:b1], hps[b0:b1], reg=reg[b0:b1], hm_hp=joints[b0:b1],
                                hp_offset=hpo[b0:b1], K=K, apply_sigmoid=sig)
        _, ws = _workspace(hm.device, b1 - b0, J, K)
        n = (b1 - b0) * (1 + J) * K
        counters = ws[2 * (-(-n * 4 // 16) * 16):].view(torch.int32)[:(b1 - b0) * J]
        assert not counters.any(), f"B = {b1 - b0}: {int(counters.count_nonzero())} pair counters left non-zero"
        return out

    got = decode(0, B, hm, hm_hp, True)
    for b in range(B):
        assert torch.equal(got[b:b + 1], decode(b, b + 1, hm, hm_hp, True)), b
    hm_s, hm_hp_s = hm.sigmoid(), hm_hp.sigmoid()
    got = decode(0, B, hm_s, hm_hp_s, False).cpu().numpy()
    for b in sorted({0, 1, B // 2, B - 1, *range(128, B, 128)}):
        inp = {k: t[b:b + 1].cpu().numpy() for k, t in
               (("heat", hm_s), ("wh", wh), ("kps", hps), ("reg", reg), ("hm_hp", hm_hp_s), ("hp_offset", hpo))}
        want = _oracle(inp, K)
        _assert_same(got[b:b + 1], want)
        assert np.array_equal(got[b:b + 1], want), b
