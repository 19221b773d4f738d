"""Device JPEG decode throughput on one GPU: ``cpb200_jpeg_decode_batch`` against ``cv2.imdecode``, and
``run_images`` from JPEG files with the device decode against the host ``cv2.imread`` (``DEVICE_PREPROCESS: false``).

    python tools/bench_jpeg.py [--images 256] [--rounds 3] [--out DIR] [--precision fp16x2] [--progressive]

The files are seeded gradients with noise (``tests/test_jpeg_cpu.make_image``) at COCO-like sizes, 640x480, 480x640
and 640x427 in turn, encoded 4:2:0 at qualities 75 and 95 in turn by ``cv2.imencode`` (with ``--progressive``, as
progressive files, ``IMWRITE_JPEG_PROGRESSIVE``), and written to ``--out`` (a temporary directory by default).

1. Decode alone.  Device: the kernels of one ``cpb200_jpeg_decode_batch`` over all images (CUDA events, median of
   ``--rounds`` launches, after a warm-up launch), and separately the host's parse + pack of the launch buffer.  Host:
   ``cv2.imdecode`` on one thread, and on a thread pool with one thread per host core (cv2 releases the GIL), over the
   same bytes.  Every device image is checked byte for byte against ``cv2.imdecode``.
2. End to end.  ``run_images(paths)`` with the DLA-34 ``dla_34`` test section, device decode against
   ``DEVICE_PREPROCESS: false``, alternated in ``--rounds`` rounds after one warm-up call of each, host clock around
   calls that end in a device-to-host copy.  The rows of the two must be identical.

The card's name, power limit and SM clocks are read before and after (nvidia-smi --query-gpu, read-only).  Prints one
JSON line.  Fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_backbones import gpu_info  # noqa: E402
from tools.bench_images import SIZES, detector  # noqa: E402
from tests.test_jpeg_cpu import encode, make_image  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the JPEG files (default: a temporary one)")
    ap.add_argument("--precision", default="fp16x2")
    ap.add_argument("--progressive", action="store_true", help="write progressive files")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_jpeg.py needs a CUDA device (there is no CPU path to time)")
    from centerpose_b200 import _lib, jpeg
    torch.cuda.set_device(0)
    out = args.out or tempfile.mkdtemp(prefix="bench_jpeg_")
    os.makedirs(out, exist_ok=True)
    datas, paths = [], []
    for i in range(args.images):
        h, w = SIZES[i % len(SIZES)]
        data = encode(make_image(h, w, "smooth_noise", 1000 + i), 75 if i % 2 == 0 else 95, "420",
                      progressive=args.progressive)
        p = os.path.join(out, "img%04d.jpg" % i)
        with open(p, "wb") as f:
            f.write(data)
        datas.append(data)
        paths.append(p)
    mb = sum(len(d) for d in datas) / 1e6
    hw_before = gpu_info(0)

    # 1. decode alone
    t0 = time.perf_counter()
    infos = [jpeg.parse(d, p) for d, p in zip(datas, paths)]
    if not all(i.eligible or i.progressive for i in infos):
        raise RuntimeError("tools/bench_jpeg.py: the device decoder does not take every file")
    sizes = [i.oh * i.ow * 3 for i in infos]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    buf, ws_bytes = jpeg.pack(infos, datas, offs[:-1])
    t_host = time.perf_counter() - t0
    src = torch.from_numpy(buf).cuda()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty(int(offs[-1]), dtype=torch.uint8, device="cuda")
    status = torch.empty(len(datas), dtype=torch.int32, device="cuda")

    def launch():
        _lib.launch("jpeg_decode_batch", src.device, src, src, len(datas), ws, ws_bytes, dst, status)

    launch()
    torch.cuda.synchronize()
    t_dev = []
    for _ in range(args.rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        launch()
        b.record()
        b.synchronize()
        t_dev.append(a.elapsed_time(b) / 1e3)
    got = dst.cpu().numpy()
    decode = lambda d: cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_COLOR)
    exact = sum(np.array_equal(got[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3), decode(d))
                for n, (i, d) in enumerate(zip(infos, datas)))
    t_one = time.perf_counter()
    for d in datas:
        decode(d)
    t_one = time.perf_counter() - t_one
    cores = os.cpu_count()
    with ThreadPoolExecutor(cores) as pool:
        list(pool.map(decode, datas))
        t_pool = time.perf_counter()
        list(pool.map(decode, datas))
        t_pool = time.perf_counter() - t_pool

    # 2. end to end from files
    det = detector("dla_34", args.precision)

    def run(device):
        det.device_preprocess = device
        return det.run_images(paths)

    rows = {True: run(True), False: run(False)}                 # warm-up: plans for every shape and batch
    times = {True: [], False: []}
    for _ in range(args.rounds):
        for device in (True, False):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows[device] = run(device)
            torch.cuda.synchronize()
            times[device].append(time.perf_counter() - t0)
    det.device_preprocess = True
    n = args.images
    result = {
        "metric": "JPEG decode images/s (device kernels vs cv2.imdecode) and run_images images/s from files",
        "images": n, "sizes_hw": SIZES, "sampling": "4:2:0", "qualities": [75, 95], "compressed_mb": round(mb, 3),
        "progressive": args.progressive,
        "device_status_ok": int((status.cpu().numpy() == 0).sum()), "device_exact_images": int(exact),
        "device_decode_images_per_s": [n / t for t in t_dev],
        "device_decode_mb_per_s": [mb / t for t in t_dev],
        "host_parse_pack_s": t_host,
        "cv2_one_thread_images_per_s": n / t_one, "cv2_one_thread_mb_per_s": mb / t_one,
        "cv2_pool_images_per_s": n / t_pool, "cv2_pool_mb_per_s": mb / t_pool, "host_cores": cores,
        "run_images_device_decode_images_per_s": [n / t for t in times[True]],
        "run_images_host_decode_images_per_s": [n / t for t in times[False]],
        "median_speedup": statistics.median(times[False]) / statistics.median(times[True]),
        "rows_identical": all(np.array_equal(a, b) for a, b in zip(rows[True], rows[False])),
        "precision": args.precision,
        "gpu_before": hw_before, "gpu_after": gpu_info(0),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
