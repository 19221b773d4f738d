"""centerpose_b200 — Hopper-native (H100, sm_90a) drop-in for the centerpose inference hot path.

Public surface mirrors the reference (tensorboy/centerpose):
  ``create_model`` / ``load_model`` / ``save_model``   (lib/models/model.py:63-131)
  ``multi_pose_decode``                                (lib/models/decode.py:235-308)
  ``detector_factory`` / ``MultiPoseDetector``         (lib/detectors/*.py)
"""
from .decode import multi_pose_decode  # noqa: F401

__version__ = "0.1.0"
