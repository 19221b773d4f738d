"""Generate the HarDNet golden fixtures by running the UNMODIFIED reference (``/root/reference``) on CPU, and pin the
oracle restatement (``oracle/hardnet_ref.py``) against it, as ``oracle/make_golden.py`` does for the other backbones.

Run:  python -m oracle.make_golden_hardnet      (from the repo root; needs /root/reference)

Writes ``tests/golden/hardnet_{128,96x160,512}.npz``: 128x128 (B=2, deepest map 2x2), 96x160 (B=2, odd pools and a
resize from a 1-pixel-high map) and 512x512 (B=1, maps subsampled at stride 4, plus the reference's decoded rows).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import hardnet_ref
from oracle.make_golden import GOLD, _ref_dets, sha
from oracle.init_recipe import conditioned_state_dict, synth_images
from oracle.ref_harness import load_reference, ref_create_model


def gen_hardnet(ns):
    model, cfg = ref_create_model("hardnet_512x512")
    sd = conditioned_state_dict(model.state_dict(), 317)
    model.load_state_dict(sd)
    sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    for tag, B, H, W, stride in (("128", 2, 128, 128, 1), ("96x160", 2, 96, 160, 1), ("512", 1, 512, 512, 4)):
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            ref = model(x)
            mine = hardnet_ref.forward(sd, x)
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"hardnet oracle != reference ({err})"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::stride, ::stride]
        extra = {"dets": _ref_dets(ns, ref, mine)} if tag == "512" else {}
        np.savez_compressed(os.path.join(GOLD, f"hardnet_{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(stride),
                            shape=np.array([B, H, W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())), **extra)
        print(f"hardnet {tag}: oracle max abs err {err:.2e} (scale {scale:.1f})")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    gen_hardnet(load_reference())
