"""Micro-benchmark of the fused decode kernel: algorithmic bytes / CUDA-event time.
Algorithmic bytes per image (SURVEY.md §8d): 1 230 848 B (read hm+hm_hp once, sparse
gathers, write the (100,56) rows)."""
import json
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import multi_pose_decode
from oracle.decode_ref import synth_decode_inputs
from bench import measured_peaks

BYTES_PER_IMG = 1230848


def main():
    peaks = measured_peaks()                  # MEASURED_PEAKS.json if present, else the H100 SXM data sheet
    print(json.dumps({"hbm_peak_gbs": peaks["hbm_gbs"], "peak_source": peaks["source"]}))
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    res = []
    sizes = [int(v) for v in os.environ.get("DECODE_BENCH_B", "32,256,1024").split(",")]
    kind = os.environ.get("DECODE_BENCH_KIND", "smooth")
    for B in sizes:
        base = synth_decode_inputs(8, 128, 128, seed=3, kind=kind)
        t = {k: torch.from_numpy(v).to(dev).repeat(B // 8, 1, 1, 1).contiguous() for k, v in base.items()}
        out = torch.empty(B, 100, 56, device=dev)
        run = lambda: multi_pose_decode(t["heat"], t["wh"], t["kps"], t["reg"], t["hm_hp"], t["hp_offset"], K=100, out=out)
        for _ in range(5):
            run()
        times = []
        for _ in range(20):
            flush.zero_()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(3_000_000)      # keep the GPU busy while the host enqueues (hides launch latency)
            e0.record(); run(); e1.record(); torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        times.sort()
        ms = times[len(times) // 2]
        gbs = B * BYTES_PER_IMG / (ms * 1e-3) / 1e9
        res.append({"B": B, "ms": ms, "min_ms": times[0], "GBps": gbs, "frac_of_hbm_peak": gbs / peaks["hbm_gbs"],
                    "peak_source": peaks["source"], "l2": "flushed"})
        print(json.dumps(res[-1]))
    return res


if __name__ == "__main__":
    main()
