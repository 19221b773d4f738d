"""Generate the MobileNetV2 and GhostNet golden fixtures by running the UNMODIFIED reference (``/root/reference``) on CPU,
and pin the oracle restatements (``oracle/mobilenetv2_ref.py``, ``oracle/ghostnet_ref.py``) against it, as
``oracle/make_golden_hardnet.py`` does for HarDNet.

Run:  python -m oracle.make_golden_mobilenetv2_ghostnet      (from the repo root; needs /root/reference)

Writes ``tests/golden/mbv2_{512,96x160}.npz`` and ``tests/golden/ghostnet_512.npz``.  Each holds the input's sha and
shape (the input is ``synth_images(B, H, W, 317)``), the conditioned weights' sha, the backbone feature and the six
head maps (concatenated on the channel axis), both subsampled every ``stride`` / ``feat_stride`` pixels, and at 512x512
the reference's decoded rows.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import ghostnet_ref, mobilenetv2_ref
from oracle.make_golden import GOLD, _ref_dets, sha
from oracle.init_recipe import conditioned_state_dict, synth_images
from oracle.ref_harness import load_reference, ref_create_model

CASES = [
    # file tag, experiments yaml, oracle, backbone function, B, H, W, map stride, feature stride
    ("mbv2_512", "mobilenetv2_512x512", mobilenetv2_ref, mobilenetv2_ref.mobilenetv2_backbone, 1, 512, 512, 4, 4),
    ("mbv2_96x160", "mobilenetv2_512x512", mobilenetv2_ref, mobilenetv2_ref.mobilenetv2_backbone, 2, 96, 160, 1, 1),
    ("ghostnet_512", "ghost_net", ghostnet_ref, ghostnet_ref.ghostnet_backbone, 1, 512, 512, 4, 8),
]


def gen(ns):
    for tag, yaml, oracle, backbone, B, H, W, st, fst in CASES:
        model, cfg = ref_create_model(yaml)
        sd = conditioned_state_dict(model.state_dict(), 317)
        model.load_state_dict(sd)
        sd_sha = sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
        x = synth_images(B, H, W, seed=317)
        with torch.no_grad():
            feat = model.backbone_model(x)
            ref = model(x)
            mine = oracle.forward(sd, x)
            mine_feat = backbone({k: v.float() for k, v in sd.items() if v.is_floating_point()}, x)
        err = max(float((a - b).abs().max()) for a, b in zip(ref, mine))
        scale = max(float(a.abs().max()) for a in ref)
        assert err <= 1e-4 * scale, f"{tag}: oracle != reference ({err})"
        assert float((feat - mine_feat).abs().max()) <= 1e-4 * float(feat.abs().max()), f"{tag}: oracle feature"
        maps = torch.cat(ref, dim=1).numpy()[:, :, ::st, ::st]
        extra = {"dets": _ref_dets(ns, ref, mine)} if H == 512 else {}
        np.savez_compressed(os.path.join(GOLD, f"{tag}.npz"), maps=maps.astype(np.float32), stride=np.array(st),
                            feat=feat.numpy()[:, :, ::fst, ::fst].astype(np.float32), feat_stride=np.array(fst),
                            shape=np.array([B, H, W]), sd_sha=np.array(sd_sha), x_sha=np.array(sha(x.numpy())), **extra)
        print(f"{tag}: oracle max abs err {err:.2e} (scale {scale:.1f}), feature {tuple(feat.shape)}")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    gen(load_reference())
