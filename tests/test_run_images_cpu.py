"""CPU tests of MultiPoseDetector.run_images' host side: the (scale, input size) grouping, and the oracle pipeline
against the reference's own run() (tests/golden/run_dla34_flip.npz, oracle/make_golden_run.py)."""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_group_by_shape_groups_splits_and_restores_order():
    from centerpose_b200.detector import group_by_shape
    keys = [(0, 256, 352), (0, 320, 224), (1, 192, 256), (0, 256, 352), (1, 192, 256), (0, 256, 352), (1, 256, 160),
            (0, 256, 352)]
    groups = group_by_shape(keys, max_batch=3)
    assert groups == [((0, 256, 352), [0, 3, 5]), ((0, 256, 352), [7]), ((0, 320, 224), [1]), ((1, 192, 256), [2, 4]),
                      ((1, 256, 160), [6])]
    for key, idx in groups:
        assert 1 <= len(idx) <= 3 and all(tuple(keys[i]) == key for i in idx)
    # every item exactly once: scattering each group's results back by index restores the input order
    out = [None] * len(keys)
    for key, idx in groups:
        for i in idx:
            assert out[i] is None
            out[i] = key
    assert out == [tuple(k) for k in keys]
    assert group_by_shape(keys, max_batch=32) == [((0, 256, 352), [0, 3, 5, 7]), ((0, 320, 224), [1]),
                                                  ((1, 192, 256), [2, 4]), ((1, 256, 160), [6])]
    assert [len(i) for _, i in group_by_shape([(0, 64, 64)] * 5, 1)] == [1] * 5
    assert group_by_shape([], 4) == []
    with pytest.raises(ValueError):
        group_by_shape(keys, 0)


def test_oracle_pipeline_reproduces_reference_run_fixture():
    """cv2 pre_process + dla_ref.forward + numpy flip merge + decode_ref + post_process_ref + the host soft_nms_39
    port, on the regenerated seeded images, vs the reference's own run() (flip, NMS, FIX_RES false; scales [1] and
    [1, 0.75])."""
    from oracle import make_golden_run as g
    from tests.util import match_rows
    f = np.load(os.path.join(GOLD, "run_dla34_flip.npz"))
    images = g.make_images()
    assert str(f["img_sha"]) == g._sha(*images), "image RNG drifted"
    sd = g.state_dict()
    assert str(f["sd_sha"]) == g._sha(*[sd[k].numpy() for k in sorted(sd) if sd[k].is_floating_point()])
    assert [tuple(s) for s in f["shapes"]] == [(h, w) for _, h, w in g.IMAGES]
    for case, scales in g.CASES.items():
        assert list(f["scales_" + case]) == scales
        for i, image in enumerate(images):
            ref = f[f"rows_{case}_{i}"]
            assert ref.shape == (100 * len(scales), 56)
            got = g.oracle_rows(sd, image, scales)
            assert got.shape == ref.shape
            rows, elems = match_rows(got, ref, tol=1e-3, box_tol=2e-2)
            assert rows >= 0.99 and elems >= 0.99, (case, i, rows, elems)
