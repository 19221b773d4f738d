"""TMA box-shape throughput (see csrc/probe.cu::probe_tma_kernel): how fast can one SM's TMA unit bring
boxes of a given shape into shared memory?  Prints GB/s (box bytes, incl. halo over-fetch) and ns per box."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import _lib

L = _lib.lib()
CASES = [
    # C, W, H, N, box_w, box_h, step_w, step_h, stages
    (64, 128, 128, 32, 16, 8, 16, 8, 4), (64, 128, 128, 32, 10, 18, 8, 16, 3), (64, 128, 128, 32, 10, 18, 8, 16, 6),
    (64, 128, 128, 32, 16, 18, 8, 16, 3), (64, 128, 128, 32, 18, 10, 16, 8, 6), (64, 128, 128, 32, 34, 6, 32, 4, 6),
    (16, 512, 512, 32, 16, 8, 16, 8, 8), (16, 512, 512, 32, 10, 18, 8, 16, 8), (16, 512, 512, 32, 34, 6, 32, 4, 8),
    (16, 512, 512, 32, 66, 4, 64, 2, 8), (16, 512, 512, 32, 130, 3, 128, 1, 8), (16, 512, 512, 32, 18, 10, 16, 8, 8),
    (32, 256, 256, 32, 10, 18, 8, 16, 8), (32, 256, 256, 32, 34, 6, 32, 4, 8),
]
for (C, W, H, N, bw, bh, sw, sh, st) in CASES:
    x = torch.zeros(N, H, W, C, dtype=torch.bfloat16, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    L.cpb200_probe_tma(x.data_ptr(), C, W, H, N, bw, bh, sw, sh, st, stream)
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = L.cpb200_probe_tma(x.data_ptr(), C, W, H, N, bw, bh, sw, sh, st, stream)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    nt = ((W + sw - 1) // sw) * ((H + sh - 1) // sh) * N
    box_bytes = C * 2 * bw * bh
    print(f"TMAPROBE C={C} map={W}x{H} box={bw}x{bh} step={sw}x{sh} stages={st}: rc={rc} {ms*1e3:8.1f} us "
          f"{nt * box_bytes / ms / 1e6:8.1f} GB/s(box bytes) {ms * 1e6 / (nt / torch.cuda.get_device_properties(0).multi_processor_count):7.1f} ns/box/SM rows/box={bw*bh}")
