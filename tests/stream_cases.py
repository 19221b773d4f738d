"""The stream table of the C ABI (tests/test_streams_gpu.py, tests/test_streams_cpu.py).  A helper module: it holds no
tests and imports without a GPU.

Every ``cpb200_*`` entry point that enqueues work takes a ``void *stream`` and must put all of it there.
``HELD`` names the cases of tests/test_streams_gpu.py and the entry points each one reaches; every case runs with its
own stream held behind a spin kernel and again with the default stream held.  ``SYNCED`` lists the wrappers that wait
for the device by design, which only take the equality leg on a side stream.  ``EXEMPT`` lists the stream-taking
entry points no case reaches, with the reason.
"""
from __future__ import annotations

import re

# the kernel families of the network program (tests/kernel_routes.py), each run in bf16 and fp16x2
PLAN_FAMILIES = ("tap", "pointwise", "halo", "small_channel", "stem", "dcn", "heads", "eltwise", "convert")

HELD = {
    **{"plan_" + f: ("run_ops",) for f in PLAN_FAMILIES},
    "model_dla34": ("run_ops",),
    "decode": ("multi_pose_decode",),
    "decode_affine": ("multi_pose_decode_affine",),
    "sigmoid": ("sigmoid_inplace",),
    "soft_nms": ("soft_nms_39",),
    "soft_nms_batch": ("soft_nms_39_batch",),
    "flip_merge": ("flip_merge",),
    "pre_process": ("pre_process",),
    "pre_process_batch": ("pre_process_batch",),
    "pre_process_batch_f32": ("pre_process_batch_f32",),
    "resize": ("resize_linear_u8_batch",),
    "jpeg": ("jpeg_decode_batch",),
    "png": ("png_decode_batch",),
    "webp": ("webp_decode_batch",),
    "webp_lossless": ("webp_lossless_decode_batch",),
    "png_encode": ("png_encode_batch",),
    "heatmap_views": ("heatmap_views_batch",),
    "render_poses": ("render_poses_batch",),
    "coco_kp_oks": ("coco_kp_oks",),
    "coco_kp_eval": ("coco_kp_eval",),
    "val_targets": ("multi_pose_targets_batch",),
    "gaussian_radius": ("gaussian_radius",),
    "val_loss": ("multi_pose_loss_batch",),
    "train_batch": ("train_augment_batch", "multi_pose_targets_train_batch"),
    "train_loss": ("multi_pose_loss_train_batch", "multi_pose_loss_train_backward"),
    "dcn_default": ("dcn_train_forward", "dcn_train_backward"),
    "dcn_fp32": ("dcn_train_forward", "dcn_train_backward"),
}

SYNCED = {
    "run_images": "reads the decode status and downloads the detections before it returns",
    "run_val": "downloads the loss stats and the detections before it returns",
    "KeypointEval.evaluate": "downloads precision, recall and scores before it returns",
}

EXEMPT = {
    "probe_halo": "hardware probe of tools/halo_probe.py, not on any product path",
    "probe_tma": "hardware probe of tools/tma_probe.py, not on any product path",
}


def stream_entry_points(text: str) -> set:
    """The names (without ``cpb200_``) of the prototypes in header ``text`` with a ``void *stream`` parameter."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^[ \t]*#[^\n]*", " ", text, flags=re.M)
    out = set()
    for stmt in re.split(r"[;{}]", text):
        m = re.fullmatch(r"(.+?)\bcpb200_(\w+)\s*\((.*)\)", stmt.strip(), re.S)
        if m and any(re.fullmatch(r"void\s*\*\s*stream", p.strip()) for p in m.group(3).split(",")):
            out.add(m.group(2))
    return out


def covered() -> set:
    return {e for entries in HELD.values() for e in entries}
