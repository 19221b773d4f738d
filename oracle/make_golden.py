"""Generate golden fixtures by running the UNMODIFIED reference (``/root/reference``) on CPU
in the build container, and pin the oracle restatements against it.

Run:  python -m oracle.make_golden            (from the repo root; needs /root/reference)

Writes small ``.npz`` fixtures into ``tests/golden/``.  Inputs are NOT stored when they can
be regenerated from a seed (``oracle.decode_ref.synth_decode_inputs``,
``oracle.init_recipe``); a sha256 of the regenerated input is stored instead so that a
silent RNG drift is detected rather than mis-reported as a parity failure.

For every fixture the script also checks the oracle restatement against the reference
output it just produced and aborts on mismatch — that is the "pinning" step required
before the oracle may be trusted as the checker for the CUDA path.
"""
from __future__ import annotations

import hashlib
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import (decode_ref, dcn_ref, dla_ref, ghostnet_ref, hardnet_ref, mobilenetv2_ref,  # noqa: E402
                    post_process_ref)
from oracle.init_recipe import conditioned_state_dict, synth_images  # noqa: E402
from oracle.ref_harness import load_reference, ref_create_model  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")

DECODE_CASES = [
    # name, B, H, W, K, kind, seed, use_reg, use_hp_offset
    ("smooth_2x128x128", 2, 128, 128, 100, "smooth", 317, True, True),
    ("uniform_1x128x128", 1, 128, 128, 100, "uniform", 318, True, True),
    ("uniform_2x96x160", 2, 96, 160, 100, "uniform", 319, True, True),
    ("smooth_1x32x40_fewpeaks", 1, 32, 40, 100, "smooth", 317, True, True),
    ("smooth_2x64x64_k50_noreg", 2, 64, 64, 50, "smooth", 5, False, False),
    ("sparse_1x64x64", 1, 64, 64, 100, "sparse", 11, True, True),
    ("lowhp_1x64x64", 1, 64, 64, 100, "lowhp", 12, True, True),
    ("uniform_1x20x12_k40_fewpeaks", 1, 20, 12, 40, "uniform", 13, True, True),
    # constructed grouping cases (decode_ref._constructed): nearest-candidate ties and the 0.1 keypoint threshold
    ("sqrttie_1x40x40", 1, 40, 40, 10, "sqrttie", 0, True, True),
    ("sqrttie_swap_1x40x40", 1, 40, 40, 10, "sqrttie_swap", 0, True, True),
    ("sqtie_1x40x40", 1, 40, 40, 10, "sqtie", 0, True, True),
    ("thresh_1x40x40", 1, 40, 40, 10, "thresh", 0, True, True),
]


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def gen_decode(ns):
    for name, B, H, W, K, kind, seed, use_reg, use_off in DECODE_CASES:
        inp = decode_ref.synth_decode_inputs(B, H, W, seed=seed, kind=kind)
        t = {k: torch.from_numpy(v.copy()) for k, v in inp.items()}
        ref = ns.multi_pose_decode(t["heat"], t["wh"], t["kps"],
                                   reg=t["reg"] if use_reg else None, hm_hp=t["hm_hp"],
                                   hp_offset=t["hp_offset"] if use_off else None, K=K).numpy()
        mine = decode_ref.multi_pose_decode(inp["heat"], inp["wh"], inp["kps"],
                                            inp["reg"] if use_reg else None, inp["hm_hp"],
                                            inp["hp_offset"] if use_off else None, K=K)
        # rows whose centre score is > 0 are tie-free by construction -> bit-exact
        pos = ref[:, :, 4] > 0
        assert np.array_equal(mine[pos], ref[pos]), f"decode oracle != reference on {name}"
        if kind not in ("sparse", "plateau") + decode_ref.CONSTRUCTED and "fewpeaks" not in name:
            assert pos.all(), name
        np.savez_compressed(os.path.join(GOLD, f"decode_{name}.npz"), det=ref,
                            meta=np.array([B, H, W, K, seed, int(use_reg), int(use_off)]),
                            kind=np.array(kind),
                            input_sha=np.array(sha(*[inp[k] for k in sorted(inp)])))
        print(f"decode {name}: {int(pos.sum())}/{pos.size} positive rows, oracle bit-exact")


def gen_dcn():
    from torchvision.ops import deform_conv2d
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 3, 6, 7, generator=g)
    off = 2.5 * torch.randn(2, 18, 6, 7, generator=g)
    msk = torch.rand(2, 9, 6, 7, generator=g)
    w = torch.randn(4, 3, 3, 3, generator=g); b = torch.randn(4, generator=g)
    tv = deform_conv2d(x, off, w, b, stride=1, padding=1, dilation=1, mask=msk).numpy()
    lit = dcn_ref.dcn_v2_forward_loops(x.numpy(), w.numpy(), b.numpy(), off.numpy(), msk.numpy())
    vec = dcn_ref.dcn_v2_forward(x, w, b, off, msk).numpy()
    assert np.abs(lit - tv).max() < 1e-5 and np.abs(vec - tv).max() < 1e-5
    np.savez_compressed(os.path.join(GOLD, "dcn_small.npz"), x=x.numpy(), off=off.numpy(),
                        msk=msk.numpy(), w=w.numpy(), b=b.numpy(), out=tv)
    print("dcn small: literal/vectorised restatements match torchvision to",
          float(np.abs(lit - tv).max()), float(np.abs(vec - tv).max()))


def gen_dla(ns):
    model, cfg = ref_create_model("dla_34_512x512")
    sd = conditioned_state_dict(model.state_dict(), 317)
    model.load_state_dict(sd)
    sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    for tag, B, H, W, stride in (("128", 1, 128, 128, 1), ("96x160", 2, 96, 160, 1), ("512", 1, 512, 512, 4)):
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = dla_ref.forward(sd, x)
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"dla oracle != reference ({err})"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::stride, ::stride]
        out = {"maps": maps.astype(np.float32), "stride": np.array(stride),
               "shape": np.array([B, H, W]), "sd_sha": np.array(sd_sha), "x_sha": np.array(sha(x.numpy()))}
        if tag == "512":
            hm, wh, hps, reg, hm_hp, hp_off = [t.clone() for t in ref]
            dets = ns.multi_pose_decode(hm.sigmoid_(), wh, hps, reg=reg, hm_hp=hm_hp.sigmoid_(),
                                        hp_offset=hp_off, K=100).numpy()
            o_in = [t.numpy() for t in mine]
            sig = lambda a: torch.from_numpy(a).sigmoid().numpy()
            dets_o = decode_ref.multi_pose_decode(sig(o_in[0]), o_in[1], o_in[2], o_in[3], sig(o_in[4]), o_in[5], K=100)
            assert np.abs(dets - dets_o).max() < 1e-3, "end-to-end oracle != reference"
            out["dets"] = dets
            meta = post_process_ref.make_meta(480, 640, 1.0, fix_res=True)
            pp = ns.multi_pose_post_process(dets.copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])
            pp = np.array(pp[0][1], dtype=np.float32).reshape(-1, 56)
            pp_o = post_process_ref.multi_pose_post_process(dets.copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])[0][1]
            assert np.abs(pp - pp_o).max() < 1e-3, float(np.abs(pp - pp_o).max())
            out["post"] = pp
        np.savez_compressed(os.path.join(GOLD, f"dla34_{tag}.npz"), **out)
        print(f"dla34 {tag}: oracle max abs err {err:.2e} (scale {scale:.1f})")



def _ref_dets(ns, ref_maps, oracle_maps):
    """Reference decode (lib/models/decode.py:235-308 after the sigmoids of lib/detectors/multi_pose.py:35-37) of the
    reference's own head maps; the oracle's decode of the oracle's maps must agree (end-to-end pin)."""
    hm, wh, hps, reg, hm_hp, hp_off = [t.clone() for t in ref_maps]
    dets = ns.multi_pose_decode(hm.sigmoid_(), wh, hps, reg=reg, hm_hp=hm_hp.sigmoid_(), hp_offset=hp_off, K=100).numpy()
    o_in = [t.numpy() for t in oracle_maps]
    sig = lambda a: torch.from_numpy(a).sigmoid().numpy()
    dets_o = decode_ref.multi_pose_decode(sig(o_in[0]), o_in[1], o_in[2], o_in[3], sig(o_in[4]), o_in[5], K=100)
    from tests.util import match_rows
    rows, elems = match_rows(dets_o[0], dets[0], tol=1e-3, box_tol=2e-2)
    assert rows >= 0.99 and elems >= 0.99, ("end-to-end oracle != reference", rows, elems)
    return dets


def gen_res50(ns):
    model, cfg = ref_create_model("res_50_512x512")
    sd = conditioned_state_dict(model.state_dict(), 317)
    model.load_state_dict(sd)
    sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    for tag, B, H, W, stride in (("128", 2, 128, 128, 1), ("512", 1, 512, 512, 4)):
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = dla_ref.forward(sd, x, arch="res_50")
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"res50 oracle != reference ({err})"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::stride, ::stride]
        extra = {"dets": _ref_dets(ns, ref, mine)} if tag == "512" else {}
        np.savez_compressed(os.path.join(GOLD, f"res50_{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(stride),
                            shape=np.array([B, H, W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())), **extra)
        print(f"res50 {tag}: oracle max abs err {err:.2e} (scale {scale:.1f})")


def gen_hrnet(ns):
    model, cfg = ref_create_model("hrnet_w32_512")
    sd = conditioned_state_dict(model.state_dict(), 317)
    model.load_state_dict(sd)
    sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    for tag, B, H, W, stride in (("128", 2, 128, 128, 1), ("256x320", 1, 256, 320, 2), ("512", 1, 512, 512, 4)):
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = dla_ref.forward(sd, x, arch="hrnet")
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"hrnet oracle != reference ({err})"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::stride, ::stride]
        extra = {"dets": _ref_dets(ns, ref, mine)} if tag == "512" else {}
        np.savez_compressed(os.path.join(GOLD, f"hrnet32_{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(stride),
                            shape=np.array([B, H, W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())), **extra)
        print(f"hrnet_w32 {tag}: oracle max abs err {err:.2e} (scale {scale:.1f})")


def gen_mbv3(ns):
    model, cfg = ref_create_model("mobilenetv3_512x512")
    sd = conditioned_state_dict(model.state_dict(), 317)
    model.load_state_dict(sd)
    sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    for tag, B, H, W, stride in (("128x160", 2, 128, 160, 1), ("512", 1, 512, 512, 4)):
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = dla_ref.forward(sd, x, arch="mobilenetv3")
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"mobilenetv3 oracle != reference ({err})"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::stride, ::stride]
        extra = {"dets": _ref_dets(ns, ref, mine)} if tag == "512" else {}
        np.savez_compressed(os.path.join(GOLD, f"mbv3_{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(stride),
                            shape=np.array([B, H, W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())), **extra)
        print(f"mobilenetv3 {tag}: oracle max abs err {err:.2e} (scale {scale:.1f})")


# One extreme-aspect input per configuration: the network input a 96x640 strip of an image becomes with TEST.FIX_RES
# false.  Its deep maps are 3x20 (1/32) and 1x10 (HarDNet's 1/64), so the product runs tensor-core tiles with fewer than
# 8 rows and maps one pixel high.  The head maps are stored every AR_STRIDE pixels (GhostNet's always-128x128 ones every 4).
AR_H, AR_W, AR_STRIDE = 96, 640, 2
AR_CASES = [
    # file tag, experiments yaml, oracle forward
    ("dla34", "dla_34_512x512", lambda sd, x: dla_ref.forward(sd, x, arch="dla_34")),
    ("res50", "res_50_512x512", lambda sd, x: dla_ref.forward(sd, x, arch="res_50")),
    ("hrnet32", "hrnet_w32_512", lambda sd, x: dla_ref.forward(sd, x, arch="hrnet")),
    ("hrnet48", "hrnet_w48_512", lambda sd, x: dla_ref.forward(sd, x, arch="hrnet")),
    ("mbv3", "mobilenetv3_512x512", lambda sd, x: dla_ref.forward(sd, x, arch="mobilenetv3")),
    ("hardnet", "hardnet_512x512", lambda sd, x: hardnet_ref.forward(sd, x)),
    ("mbv2", "mobilenetv2_512x512", lambda sd, x: mobilenetv2_ref.forward(sd, x)),
    ("ghostnet", "ghost_net", lambda sd, x: ghostnet_ref.forward(sd, x)),
]


def gen_aspect(ns):
    for name, yaml, oracle in AR_CASES:
        model, cfg = ref_create_model(yaml)
        sd = conditioned_state_dict(model.state_dict(), 317)
        model.load_state_dict(sd)
        sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
        x = synth_images(1, AR_H, AR_W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = oracle(sd, x)
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"{name} {AR_H}x{AR_W}: oracle != reference ({err})"
        st = 4 if ref[0].shape[2] == 128 else AR_STRIDE
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::st, ::st]
        tag = f"{name}_{AR_H}x{AR_W}"
        np.savez_compressed(os.path.join(GOLD, f"{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(st),
                            shape=np.array([1, AR_H, AR_W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())))
        print(f"{tag}: oracle max abs err {err:.2e} (scale {scale:.1f}), maps {tuple(ref[0].shape[2:])}")


def gen_soft_nms(ns=None):
    """Golden vectors of the reference's own Cython ``soft_nms_39`` compiled here (oracle/build_ref.py)."""
    from oracle.build_ref import load
    from centerpose_b200.soft_nms import soft_nms_39
    nms = load()
    assert nms is not None, "reference tree absent"
    rng = np.random.RandomState(39)
    ins, outs, keeps, params = [], [], [], []
    for trial in range(24):
        N = int(rng.randint(1, 100))
        c = rng.uniform(0, 400, size=(N, 2)); wh = rng.uniform(5, 200, size=(N, 2))
        rows = np.zeros((100, 56), np.float32)
        rows[:N, 0:2] = c - wh / 2; rows[:N, 2:4] = c + wh / 2; rows[:N, 4] = rng.uniform(0, 1, N)
        if trial % 4 == 0:
            rows[:N, 4] = np.round(rows[:N, 4], 1)                         # score ties
        rows[:N, 5:] = rng.uniform(0, 400, size=(N, 51))
        method, Nt, thr = trial % 3, (0.3, 0.5, 0.7)[trial % 3], (0.001, 0.05)[trial % 2]
        a = rows[:N].copy(); b = rows[:N].copy()
        ka = nms.soft_nms_39(a, sigma=0.5, Nt=Nt, threshold=thr, method=method)
        kb = soft_nms_39(b, sigma=0.5, Nt=Nt, threshold=thr, method=method)
        assert list(ka) == list(kb), (trial, len(ka), len(kb))
        assert np.abs(a - b).max() <= 2e-7, float(np.abs(a - b).max())     # 1 ulp of a score in (0,1]: see test
        out = np.zeros((100, 56), np.float32); out[:N] = a
        ins.append(rows); outs.append(out); keeps.append(len(ka)); params.append([N, method, Nt, thr])
    np.savez_compressed(os.path.join(GOLD, "soft_nms.npz"), boxes=np.stack(ins), out=np.stack(outs),
                        keep=np.array(keeps), params=np.array(params, np.float64))
    print("soft_nms_39: port == compiled reference on 24 cases (keep lists equal, scores within 1 ulp)")


def gen_soft_nms_cases(ns=None):
    """The reference's own Cython ``soft_nms_39`` (oracle/build_ref.py) on the constructed soft-NMS cases of
    tests/post_cases.py; the inputs are rebuilt from the cases, so only their sha256 is stored."""
    from oracle.build_ref import load
    from tests import post_cases as pc
    from tests.test_post_cases_cpu import assert_matches_cython
    nms = load()
    assert nms is not None, "reference tree absent"
    store = {}
    for case in pc.NMS_CASES:
        rows = case.build()
        out = rows.copy()
        keep = len(nms.soft_nms_39(out, **case.params()))
        store[f"out_{case.label}"] = out
        store[f"keep_{case.label}"] = np.array(keep)
        store[f"sha_{case.label}"] = np.array(pc.digest(rows))
    for case in pc.NMS_CASES:                  # pin: the port agrees with what was just stored
        port = case.build()
        k = pc.soft_nms_literal(port, **case.params())
        assert_matches_cython(port, k, store, case)
    np.savez_compressed(os.path.join(GOLD, "soft_nms_cases.npz"), **store)
    print(f"soft_nms_39: {len(pc.NMS_CASES)} constructed cases, port == compiled reference (keeps and moves exact, "
          "scores within 1 ulp)")


def gen_post(ns):
    rng = np.random.RandomState(3)
    dets = rng.uniform(0, 128, size=(1, 100, 56)).astype(np.float32)
    cases = []
    for (h, w, scale, fix) in ((480, 640, 1.0, True), (427, 640, 1.0, False), (333, 500, 0.75, False), (1080, 1920, 1.0, True)):
        meta = post_process_ref.make_meta(h, w, scale, fix_res=fix)
        ref = ns.multi_pose_post_process(dets.copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])
        ref = np.array(ref[0][1], dtype=np.float32).reshape(-1, 56)
        mine = post_process_ref.multi_pose_post_process(dets.copy(), [meta["c"]], [meta["s"]], meta["out_height"], meta["out_width"])[0][1]
        err = float(np.abs(ref - mine).max())
        assert err < 2e-3, err
        cases.append(ref)
        print(f"post_process {h}x{w} scale {scale} fix_res {fix}: oracle err {err:.2e}")
    np.savez_compressed(os.path.join(GOLD, "post_process.npz"), dets=dets, out=np.stack(cases),
                        cases=np.array([[480, 640, 1.0, 1], [427, 640, 1.0, 0], [333, 500, 0.75, 0], [1080, 1920, 1.0, 1]]))


def gen_flip(ns):
    g = torch.Generator().manual_seed(9)
    hm_hp = torch.rand(1, 17, 8, 12, generator=g); hps = torch.randn(1, 34, 8, 12, generator=g)
    idx = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    np.savez_compressed(os.path.join(GOLD, "flip.npz"), hm_hp=hm_hp.numpy(), hps=hps.numpy(),
                        flip_tensor=ns.flip_tensor(hm_hp).numpy(), flip_lr=ns.flip_lr(hm_hp, idx).numpy(),
                        flip_lr_off=ns.flip_lr_off(hps, idx).numpy())
    print("flip helpers stored")


def main():
    os.makedirs(GOLD, exist_ok=True)
    ns = load_reference()
    if len(sys.argv) > 1:                       # python -m oracle.make_golden hrnet  -> only that family
        for name in sys.argv[1:]:
            globals()["gen_" + name](ns) if name not in ("dcn",) else gen_dcn()
        return
    gen_decode(ns)
    gen_dcn()
    gen_post(ns)
    gen_flip(ns)
    gen_dla(ns)
    gen_res50(ns)
    gen_hrnet(ns)
    gen_mbv3(ns)
    gen_aspect(ns)
    gen_soft_nms(ns)
    gen_soft_nms_cases(ns)
    print("golden fixtures written to", GOLD)


if __name__ == "__main__":
    main()
