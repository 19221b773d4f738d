"""Device WebP decode throughput on one GPU: ``cpb200_webp_decode_batch`` against ``cv2.imdecode``, and
``run_images`` from lossy WebP files with the device decode against the host ``cv2.imread`` (``DEVICE_PREPROCESS:
false``).

    python tools/bench_webp.py [--images 256] [--batches 1,16,32,64,128,256] [--counts 1,4,16,64,256] [--rounds 3]
                               [--out DIR] [--precision fp16x2]

The images are seeded gradients with noise (``tests/test_jpeg_cpu.make_image``) at COCO-like sizes, 640x480, 480x640
and 640x427 in turn, written lossy by ``cv2.imencode`` at quality 75 and at quality 95.  Each set goes to ``--out`` (a
temporary directory by default).

1. Decode alone, per set and per batch size in ``--batches``.  Device: the kernels of one ``cpb200_webp_decode_batch``
   over the first ``batch`` images (CUDA events, median of ``--rounds`` launches after a warm-up launch).  Host:
   ``cv2.imdecode`` on one thread, and on a thread pool with one thread per host core (cv2 releases the GIL), over all
   the set's bytes.  Every device image is checked byte for byte against ``cv2.imdecode``.
2. End to end, quality-75 set, on the first n files for each n in ``--counts``, with ``WEBP_DEVICE_MIN_IMAGES`` set
   to 1 so that every call decodes on the device.  ``run_images(paths)`` with the DLA-34 ``dla_34`` test section,
   device decode against ``DEVICE_PREPROCESS: false``, alternated in ``--rounds`` rounds after one warm-up call of
   each, host clock around calls that end in a device-to-host copy.  The rows of the two must be identical.

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
from tests.test_jpeg_cpu import make_image  # noqa: E402


def _files(quality, n, out):
    datas, paths = [], []
    for i in range(n):
        h, w = SIZES[i % len(SIZES)]
        im = make_image(h, w, "smooth_noise", 1000 + i)
        data = cv2.imencode(".webp", im, [cv2.IMWRITE_WEBP_QUALITY, quality])[1].tobytes()
        p = os.path.join(out, "q%d_%04d.webp" % (quality, i))
        with open(p, "wb") as f:
            f.write(data)
        datas.append(data)
        paths.append(p)
    return datas, paths


def _decode_alone(datas, batches, rounds):
    from centerpose_b200 import _lib, webp
    decode = lambda d: cv2.imdecode(np.frombuffer(d, np.uint8), cv2.IMREAD_COLOR)
    res = {"compressed_mb": round(sum(len(d) for d in datas) / 1e6, 3), "device": {}}
    exact = 0
    for B in batches:
        sub = datas[:B]
        t0 = time.perf_counter()
        infos = [webp.parse(d) for d in sub]
        sizes = [i.oh * i.ow * 3 for i in infos]
        offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        buf, ws_bytes = webp.pack(infos, sub, offs[:-1])
        t_host = time.perf_counter() - t0
        src = torch.from_numpy(buf).cuda()
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        dst = torch.empty(int(offs[-1]), dtype=torch.uint8, device="cuda")
        status = torch.empty(len(sub), dtype=torch.int32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def launch():
            _lib.check(_lib.lib().cpb200_webp_decode_batch(src.data_ptr(), src.data_ptr(), len(sub), ws.data_ptr(),
                                                           ws_bytes, dst.data_ptr(), status.data_ptr(), stream),
                       "webp_decode_batch")

        launch()
        torch.cuda.synchronize()
        t_dev = []
        for _ in range(rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            launch()
            b.record()
            b.synchronize()
            t_dev.append(a.elapsed_time(b) / 1e3)
        if B == max(batches):
            got = dst.cpu().numpy()
            exact = sum(np.array_equal(got[offs[n]:offs[n + 1]].reshape(i.oh, i.ow, 3), decode(d))
                        for n, (i, d) in enumerate(zip(infos, sub)))
            res["device_status_ok"] = int((status.cpu().numpy() == 0).sum())
        res["device"][B] = {"images_per_s": B / statistics.median(t_dev), "launch_ms": [t * 1e3 for t in t_dev],
                            "host_parse_pack_s": t_host}
    res["device_exact_images"] = int(exact)
    t_one = time.perf_counter()
    for d in datas:
        decode(d)
    t_one = time.perf_counter() - t_one
    with ThreadPoolExecutor(os.cpu_count()) as pool:
        list(pool.map(decode, datas))
        t_pool = time.perf_counter()
        list(pool.map(decode, datas))
        t_pool = time.perf_counter() - t_pool
    res["cv2_one_thread_images_per_s"] = len(datas) / t_one
    res["cv2_pool_images_per_s"] = len(datas) / t_pool
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--batches", default="1,16,32,64,128,256")
    ap.add_argument("--counts", default="1,4,16,64,256")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the WebP files (default: a temporary one)")
    ap.add_argument("--precision", default="fp16x2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_webp.py needs a CUDA device (there is no CPU path to time)")
    torch.cuda.set_device(0)
    out = args.out or tempfile.mkdtemp(prefix="bench_webp_")
    os.makedirs(out, exist_ok=True)
    batches = sorted({min(int(b), args.images) for b in args.batches.split(",")})
    hw_before = gpu_info(0)
    sets, decode = {}, {}
    for quality in (75, 95):
        sets[quality] = _files(quality, args.images, out)
        decode["q%d" % quality] = _decode_alone(sets[quality][0], batches, args.rounds)

    from centerpose_b200 import detector as detector_mod
    det = detector("dla_34", args.precision)
    detector_mod.WEBP_DEVICE_MIN_IMAGES = 1
    e2e = {}
    for n in sorted({min(int(c), args.images) for c in args.counts.split(",")}):
        paths = sets[75][1][:n]

        def run(device):
            det.device_preprocess = device
            return det.run_images(paths)

        rows = {True: run(True), False: run(False)}             # warm-up: plans for every shape and batch
        times = {True: [], False: []}
        for _ in range(args.rounds):
            for device in (True, False):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rows[device] = run(device)
                torch.cuda.synchronize()
                times[device].append(time.perf_counter() - t0)
        e2e[n] = {"device_decode_images_per_s": [n / t for t in times[True]],
                  "host_decode_images_per_s": [n / t for t in times[False]],
                  "median_speedup": statistics.median(times[False]) / statistics.median(times[True]),
                  "rows_identical": all(np.array_equal(a, b) for a, b in zip(rows[True], rows[False]))}
    det.device_preprocess = True
    result = {
        "metric": "lossy WebP decode images/s (device kernels vs cv2.imdecode) and run_images images/s from files",
        "images": args.images, "sizes_hw": SIZES, "host_cores": os.cpu_count(), "decode": decode,
        "run_images_set": "q75", "run_images": e2e,
        "precision": args.precision,
        "gpu_before": hw_before, "gpu_after": gpu_info(0),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
