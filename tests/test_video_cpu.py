"""CPU tests of run_video's host side: the frame source (centerpose_b200.video.FrameReader), its frame order and content
against a plain ``cv2.VideoCapture`` loop on videos written here (``mp4v`` .mp4, ``MJPG`` .avi) and on iterables, the
bound on the buffer ring, shape groups, the end of a stream, errors raised in the caller's thread and the reader
thread's teardown; the ellipse2Poly model (tests/ellipse_model.py) against cv2 over its exhaustive domain; the
prototypes of include/centerpose_b200_video.h and its stream cases."""
import ctypes
import re
import threading
import time

import cv2
import numpy as np
import pytest

from centerpose_b200.video import FrameReader, is_live


def frame(h, w, i):
    """A frame whose content says its index: a bar at a row that moves and a level that changes per frame."""
    im = np.empty((h, w, 3), np.uint8)
    im[:] = ((i * 37) % 256, (i * 11 + 60) % 256, (200 - i * 5) % 256)
    im[(i * 3) % h] = 255
    im[:, (i * 5) % w] = 0
    return im


def write_video(path, fourcc, n, h, w, fps=25):
    vw = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*fourcc), fps, (w, h))
    assert vw.isOpened(), path
    for i in range(n):
        vw.write(frame(h, w, i))
    vw.release()
    return str(path)


def capture_frames(path):
    """tools/demo.py's read loop, up to the first failed read."""
    cap = cv2.VideoCapture(path)
    out = []
    while True:
        ok, im = cap.read()
        if not ok:
            break
        out.append(im)
    cap.release()
    return out


def reader_threads():
    return [t for t in threading.enumerate() if t.name == "FrameReader"]


def collect(reader):
    out = []
    for fr in reader:
        out.append((fr.index, fr.image.copy()))
        fr.release()
    return out


@pytest.mark.parametrize("fourcc,ext", [("mp4v", "mp4"), ("MJPG", "avi")])
@pytest.mark.parametrize("slots", [1, 3, 16])
def test_video_frames_equal_capture_loop(tmp_path, fourcc, ext, slots):
    path = write_video(tmp_path / ("v." + ext), fourcc, 13, 48, 64)
    want = capture_frames(path)
    assert len(want) == 13
    got = collect(FrameReader(path, slots=slots))
    assert [i for i, _ in got] == list(range(len(want)))
    for (_, g), w in zip(got, want):
        assert g.dtype == np.uint8 and np.array_equal(g, w)
    assert not reader_threads()


def test_iterable_order_and_shape_groups():
    shapes = [(20, 30)] * 3 + [(31, 17)] * 2 + [(20, 30)] + [(5, 7)] * 4
    frames = [frame(h, w, i) for i, (h, w) in enumerate(shapes)]
    got = collect(FrameReader(iter(frames), slots=2))
    assert [i for i, _ in got] == list(range(len(frames)))
    for (_, g), w in zip(got, frames):
        assert g.shape == w.shape and np.array_equal(g, w)
    assert not reader_threads()


def test_ring_is_bounded():
    """With every frame held, the reader reads one frame past the ring and waits; each release lets one more in, and
    no more than ``slots`` buffers ever exist."""
    pulled = []

    def source():
        for i in range(20):
            pulled.append(i)
            yield frame(8, 8, i)

    reader = FrameReader(source(), slots=4)
    it = iter(reader)
    held = [next(it) for _ in range(4)]
    time.sleep(0.3)
    assert len(pulled) <= 5
    assert reader._out.qsize() == 0
    held.pop(0).release()
    held.append(next(it))
    time.sleep(0.3)
    assert len(pulled) <= 6
    buffers = {fr.slot.data_ptr() for fr in held}
    while True:
        held.pop(0).release()
        fr = next(it, None)
        if fr is None:
            break
        buffers.add(fr.slot.data_ptr())
        held.append(fr)
    assert len(buffers) <= 4
    assert len(pulled) == 20
    assert [fr.index for fr in held] == [17, 18, 19]
    assert not reader_threads()


def test_end_of_stream():
    assert collect(FrameReader([], slots=2)) == []
    assert len(collect(FrameReader([frame(4, 4, 0)]))) == 1
    assert not reader_threads()


def test_video_without_frames_yields_nothing(tmp_path):
    path = str(tmp_path / "empty.avi")
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 25, (64, 48))
    vw.release()
    try:
        reader = FrameReader(path)
    except FileNotFoundError:
        return                                   # this cv2 build does not open a video without frames
    assert collect(reader) == []
    assert not reader_threads()


def test_truncated_video_ends_cleanly(tmp_path):
    """A read that fails part-way ends the stream after the frames before it, as the capture loop stops there."""
    path = write_video(tmp_path / "v.avi", "MJPG", 12, 48, 64)
    data = open(path, "rb").read()
    cut = str(tmp_path / "cut.avi")
    with open(cut, "wb") as f:
        f.write(data[:len(data) * 2 // 3])
    want = capture_frames(cut)
    got = collect(FrameReader(cut))
    assert len(got) == len(want)
    for (_, g), w in zip(got, want):
        assert np.array_equal(g, w)
    assert not reader_threads()


def test_missing_path_raises_before_reading(tmp_path):
    with pytest.raises(FileNotFoundError):
        FrameReader(str(tmp_path / "nope.mp4"))
    assert not reader_threads()


def test_reader_errors_reach_the_caller():
    def source():
        yield frame(6, 6, 0)
        yield frame(6, 6, 1)
        raise KeyError("camera unplugged")

    it = iter(FrameReader(source()))
    assert [next(it).index, next(it).index] == [0, 1]
    with pytest.raises(KeyError, match="unplugged"):
        next(it)
    assert not reader_threads()
    for bad in (np.zeros((4, 4), np.uint8), np.zeros((4, 4, 3), np.float32), "frame.png"):
        with pytest.raises(ValueError, match="frame 1 must be"):
            collect(FrameReader([frame(4, 4, 0), bad]))
        assert not reader_threads()
    with pytest.raises(ValueError, match="source must be"):
        FrameReader(3.5)


def test_thread_is_joined_on_every_exit(tmp_path):
    path = write_video(tmp_path / "v.avi", "MJPG", 30, 48, 64)
    # close() part-way, with the reader blocked on a full ring
    reader = FrameReader(path, slots=2)
    it = iter(reader)
    next(it), next(it)
    time.sleep(0.2)
    assert reader_threads()
    reader.close()
    assert not reader_threads()
    # the generator closed by the caller
    it = iter(FrameReader(path, slots=2))
    next(it)
    it.close()
    assert not reader_threads()
    # an exception in the caller's loop
    with pytest.raises(RuntimeError, match="caller"):
        with FrameReader(path, slots=2) as reader:
            for fr in reader:
                raise RuntimeError("caller")
    assert not reader_threads()
    # a reader is iterated once
    reader = FrameReader([frame(4, 4, 0)])
    collect(reader)
    with pytest.raises(RuntimeError, match="once"):
        collect(reader)


def test_live_sources():
    assert is_live("webcam") and is_live(0) and is_live(np.int64(2))
    assert not (is_live("clip.mp4") or is_live(True) or is_live([np.zeros((2, 2, 3), np.uint8)]))


def test_ellipse_model_matches_cv2_exhaustively():
    """Every integer angle in [-180, 180], every half-length up to a 4096 x 4096 frame's longest limb, two centres of
    opposite parities: the model's points are cv2.ellipse2Poly's, point for point."""
    from tests import ellipse_model as em
    cx, cy, L = em.domain()
    for angle in range(-180, 181):
        pts, counts = em.ellipse_polys(cx, cy, L, angle)
        want = [cv2.ellipse2Poly((int(x), int(y)), (int(l), 2), angle, 0, 360, 1) for x, y, l in zip(cx, cy, L)]
        assert np.array_equal(counts, [len(p) for p in want]), angle
        assert np.array_equal(pts, np.concatenate(want).reshape(-1, 2)), angle


def _video_header():
    from centerpose_b200 import _lib
    with open(_lib.VIDEO_HEADER) as f:
        return f.read()


def test_video_prototypes_bind():
    """The prototypes of include/centerpose_b200_video.h parse, are exported and are bound as declared."""
    from centerpose_b200 import _lib
    text = _video_header()
    sigs = _lib.signatures(text)
    code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    assert set(sigs) == set(re.findall(r"\b(cpb200_[a-z0-9_]+)\s*\(", code))
    assert set(sigs) == {"cpb200_ellipse_poly_batch", "cpb200_render_plan_batch"}
    assert not set(sigs) & set(_lib.signatures()), "declared in two public headers"
    I, P, I64 = ctypes.c_int, ctypes.c_void_p, ctypes.c_int64
    assert sigs["cpb200_ellipse_poly_batch"] == (I, [P, I, P, P, P])
    assert sigs["cpb200_render_plan_batch"] == (I, [P, I, I, I, I, ctypes.c_double, I, P, I, I64, I64] + [P] * 7)
    assert _lib.VIDEO_HEADER in _lib.HEADERS
    L = _lib.lib()
    for n, (restype, argtypes) in sigs.items():
        fn = getattr(L, n)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, n


def test_every_video_stream_entry_point_has_a_stream_case():
    """Every entry point of the video header that takes a stream is held on a side stream by a case of
    tests/test_video_streams_gpu.py, and the stream is its last parameter, as _lib.launch appends it."""
    from centerpose_b200 import _lib
    from tests.stream_cases import stream_entry_points
    from tests.video_cases import STREAM_CASES
    declared = stream_entry_points(_video_header())
    covered = {e for entries in STREAM_CASES.values() for e in entries}
    assert declared == covered, (sorted(declared), sorted(covered))
    sigs = _lib.signatures(_video_header())
    for name in declared:
        assert sigs["cpb200_" + name][1][-1] is ctypes.c_void_p, name


def test_label_table_and_strings():
    """Label index k is the text "{:.1f}" gives every score that rounds to k / 10; the metrics are cv2's."""
    from centerpose_b200 import render
    for k in range(render.LABELS):
        for score in (k / 10, k / 10 + 0.0499, max(k / 10 - 0.05 + 1e-9, 0.0)):
            assert render.label_text(score) == render.label_string(k), (k, score)
    t = render.label_table(render.LABELS)
    for k in range(render.LABELS):
        (tw, th), _ = cv2.getTextSize(render.label_string(k), render.FONT, 0.5, 2)
        assert (t[k]["tw"], t[k]["th"]) == (tw, th)


def test_device_plan_refuses_negative_threshold():
    from centerpose_b200 import render
    with pytest.raises(ValueError, match="VIS_THRESH"):
        render.DevicePlan(-0.1, "white", None)
