"""Frame source of ``MultiPoseDetector.run_video``: the video and webcam branch of the reference's ``tools/demo.py``
(``cv2.VideoCapture`` read frame by frame) with the decode moved to a background thread.

``FrameReader(source)`` reads a video path (``cv2.VideoCapture(path)``, its default backend, as tools/demo.py),
``"webcam"`` or a camera index (``cv2.VideoCapture(index)``), or any iterable of BGR uint8 (H, W, 3) arrays.  A
thread decodes the frames into a ring of at most ``slots`` host buffers, pinned when CUDA is available so that a
frame's upload is an asynchronous copy.  The buffers are sized from the first frame; a frame of another size (an
iterable only: a video keeps one size) starts a new shape group, and the buffers of the old size are dropped as they
come back, so at most ``slots`` buffers exist at any time.

Iterating yields ``Frame`` objects in frame order.  A frame's buffer returns to the ring when the caller calls
``Frame.release()``; until then the reader may be ``slots`` frames ahead and no further.

Differences from tools/demo.py, on purpose:
  * a path that does not open (``cv2.VideoCapture.isOpened()`` false) raises ``FileNotFoundError``;
  * a failed ``read()`` ends the stream: the frames before it are yielded and no more (tools/demo.py hands the
    ``None`` frame to ``detector.run`` and crashes there);
  * a stream with no frames yields nothing.
An error in the reader thread (an iterable that raises, a frame that is not uint8 (H, W, 3)) is raised in the caller's
thread when the frames before it are consumed.  The thread is joined when the iteration ends: at the last frame, on
``close()``, on an exception in the caller, or when the generator is closed or collected.
"""
from __future__ import annotations

import queue
import threading
from dataclasses import dataclass

import cv2
import numpy as np
import torch

VIDEO_EXTENSIONS = ("mp4", "mov", "avi", "mkv")       # the extensions tools/demo.py reads with cv2.VideoCapture
_POLL_S = 0.05


def is_live(source):
    """True for the sources tools/demo.py treats as a camera: ``"webcam"`` or a camera index."""
    if isinstance(source, str):
        return source == "webcam"
    return isinstance(source, (int, np.integer)) and not isinstance(source, bool)


@dataclass
class Frame:
    index: int
    image: np.ndarray          # (H, W, 3) uint8 BGR, a view of the slot
    slot: torch.Tensor         # the (H * W * 3,) uint8 host buffer the image lives in
    _reader: "FrameReader"

    def release(self):
        """Hands the frame's buffer back to the reader; ``image`` must not be used after this."""
        if self._reader is not None:
            self._reader._release(self.slot)
            self._reader = None


class _End:
    pass


class FrameReader:
    def __init__(self, source, slots=8):
        if int(slots) < 1:
            raise ValueError("FrameReader: slots must be >= 1, got %r" % (slots,))
        self.slots = int(slots)
        self._cap = None
        self._iter = None
        if isinstance(source, str) and source != "webcam":
            self._cap = cv2.VideoCapture(source)
            if not self._cap.isOpened():
                self._cap.release()
                raise FileNotFoundError(source)
        elif is_live(source):
            index = 0 if source == "webcam" else int(source)
            self._cap = cv2.VideoCapture(index)
            if not self._cap.isOpened():
                self._cap.release()
                raise FileNotFoundError("camera %d does not open" % index)
        else:
            try:
                self._iter = iter(source)
            except TypeError:
                raise ValueError("FrameReader: source must be a video path, 'webcam', a camera index or an iterable of "
                                 "BGR uint8 (H, W, 3) arrays, got %s" % type(source).__name__) from None
        self.live = is_live(source)
        self._pin = torch.cuda.is_available()
        self._out = queue.Queue()
        self._free = queue.Queue()                # released buffers
        self._room = threading.Semaphore(self.slots)
        self._stop = threading.Event()
        self._thread = None
        self._started = False

    # -- reader thread ------------------------------------------------------------------------------
    def _slot(self, nbytes):
        """A buffer of ``nbytes`` for the next frame, once fewer than ``slots`` frames are out.  None when stopped."""
        while not self._room.acquire(timeout=_POLL_S):
            if self._stop.is_set():
                return None
        while True:
            try:
                buf = self._free.get_nowait()
            except queue.Empty:
                break
            if buf.numel() == nbytes:
                return buf
            # a buffer of the previous shape group: dropped
        return torch.empty(nbytes, dtype=torch.uint8, pin_memory=self._pin)

    def _next_image(self, buf_view):
        """The next frame, or None at the end.  A capture decodes into ``buf_view`` when it can."""
        if self._cap is not None:
            ok, image = self._cap.read() if buf_view is None else self._cap.read(buf_view)
            return image if ok and image is not None else None
        try:
            image = next(self._iter)
        except StopIteration:
            return None
        return image

    def _run(self):
        try:
            shape, n = None, 0
            while not self._stop.is_set():
                buf = None
                if self._cap is not None and shape is not None:
                    buf = self._slot(int(np.prod(shape)))
                    if buf is None:
                        break
                image = self._next_image(None if buf is None else buf.numpy().reshape(shape))
                if image is None:
                    if buf is not None:
                        self._release(buf)
                    break
                if not (isinstance(image, np.ndarray) and image.dtype == np.uint8 and image.ndim == 3
                        and image.shape[2] == 3):
                    raise ValueError("FrameReader: frame %d must be a BGR uint8 (H, W, 3) array, got %s" % (
                        n, "%s %s" % (image.dtype, image.shape) if isinstance(image, np.ndarray)
                        else type(image).__name__))
                if buf is None or tuple(image.shape) != shape:
                    if buf is not None:
                        self._release(buf)
                    shape = tuple(image.shape)
                    buf = self._slot(image.nbytes)
                    if buf is None:
                        break
                view = buf.numpy().reshape(shape)
                if view.__array_interface__["data"][0] != image.__array_interface__["data"][0]:
                    view[...] = image
                self._out.put(Frame(n, view, buf, self))
                n += 1
        except BaseException as e:                   # raised in the caller's thread, after the frames before it
            self._out.put(e)
        finally:
            self._out.put(_End)

    def _release(self, buf):
        self._free.put(buf)
        self._room.release()

    # -- caller side --------------------------------------------------------------------------------
    def __iter__(self):
        if self._started:
            raise RuntimeError("FrameReader: a reader is iterated once")
        self._started = True
        self._thread = threading.Thread(target=self._run, name="FrameReader", daemon=True)
        self._thread.start()
        try:
            while True:
                item = self._out.get()
                if item is _End:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            self.close()

    def close(self):
        """Stops and joins the reader thread and releases the capture.  Safe to call more than once."""
        self._stop.set()
        if self._thread is not None:
            while self._thread.is_alive():
                # the thread may wait for room: unblock it by draining what it queued
                try:
                    item = self._out.get(timeout=_POLL_S)
                    if isinstance(item, Frame):
                        item.release()
                except queue.Empty:
                    pass
            self._thread.join()
            self._thread = None
        if self._cap is not None:
            self._cap.release()
            self._cap = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
