"""Video throughput in frames/s: MultiPoseDetector.run_video against tools/demo.py's loop of run(frame) per
cv2.VideoCapture frame, against run_images on chunks of max_batch decoded frames, and against the host decode alone
(the cv2.VideoCapture read loop).  Each with and without return_images (run()'s drawing is render_poses per frame),
on seeded 640x480 and 1280x720 mp4v videos written to a temporary directory, DLA-34 in fp16x2 with the conditioned
weights and the dla_34 test section.  Three alternated rounds; every round's outputs must equal the first round's, and
run_video's must equal run_images'.  Prints the card and its power limit.

The run() loop is timed on the first --loop-frames frames only (its rate does not depend on the clip's length).

    python tools/bench_video.py [--frames 512] [--loop-frames 128] [--rounds 3] [--max-batch 32]
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
import time

import cv2
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import render_cases as rc  # noqa: E402
from tools.bench_images import detector  # noqa: E402
from tools.bench_render import card  # noqa: E402

SHAPES = [(480, 640), (720, 1280)]


def write_video(path, n, h, w):
    """A seeded clip: a smooth background that drifts frame to frame (mp4v at 25 fps)."""
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 25, (w, h))
    base = rc.image(h, w, 7)
    for i in range(n):
        vw.write(np.roll(base, (i * 3) % w, axis=1))
    vw.release()


def host_decode(path):
    cap = cv2.VideoCapture(path)
    out = []
    while True:
        ok, im = cap.read()
        if not ok:
            break
        out.append(im)
    cap.release()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=32)
    ap.add_argument("--loop-frames", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_video needs a CUDA device")
    det = detector("dla_34", "fp16x2")
    mb = args.max_batch
    print("card:", card())
    with tempfile.TemporaryDirectory() as tmp:
        for h, w in SHAPES:
            path = os.path.join(tmp, "clip_%dx%d.mp4" % (w, h))
            write_video(path, args.frames, h, w)
            n = len(host_decode(path))
            for draw in (False, True):
                def run_video():
                    return list(det.run_video(path, max_batch=mb, return_images=draw))

                def run_loop():
                    out = []
                    for i, frame in enumerate(host_decode(path)[:args.loop_frames]):
                        rows = np.asarray(det.run(frame)["results"][1], np.float32)
                        out.append((i, rows, det.render_poses([frame], [rows])[0]) if draw else (i, rows))
                    return out

                def run_images():
                    frames, out = host_decode(path), []
                    for a in range(0, len(frames), mb):
                        res = det.run_images(frames[a:a + mb], max_batch=mb, return_images=draw)
                        rows = res[0] if draw else res
                        for k in range(len(rows)):
                            out.append((a + k, rows[k], res[1][k]) if draw else (a + k, rows[k]))
                    return out

                ways = {"run_video": run_video, "run() loop": run_loop, "run_images chunks": run_images,
                        "host decode": lambda: host_decode(path)}
                times = {k: [] for k in ways}
                first = {}
                for r in range(args.rounds):
                    for name, fn in ways.items():
                        torch.cuda.synchronize()
                        t = time.perf_counter()
                        out = fn()
                        torch.cuda.synchronize()
                        times[name].append(time.perf_counter() - t)
                        if name not in first:
                            first[name] = out
                        else:
                            same = all(all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))
                                       for a, b in zip(out, first[name])) if name != "host decode" else \
                                all(np.array_equal(x, y) for x, y in zip(out, first[name]))
                            assert len(out) == len(first[name]) and same, (name, r)
                for a, b in zip(first["run_video"], first["run_images chunks"]):
                    assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:])), a[0]
                for name, ts in times.items():
                    m = min(n, args.loop_frames) if name == "run() loop" else n
                    print("%dx%d %-18s return_images=%-5s %7.1f frames/s (best of %d, %d frames)"
                          % (w, h, name, draw, m / min(ts), len(ts), m), flush=True)


if __name__ == "__main__":
    main()
