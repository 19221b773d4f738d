"""Run the wgmma halo-descriptor probe (see csrc/probe.cu) and report which variant is exact."""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import _lib

L = _lib.lib()
g = torch.Generator().manual_seed(1)
x = torch.randint(-4, 5, (1, 64, 18, 10), generator=g).float()
w = torch.randint(-2, 3, (64, 64, 3, 3), generator=g).float()
ref = F.conv2d(x, w)                                   # valid conv: (1,64,16,8)
ref = ref[0].permute(1, 2, 0).reshape(128, 64)
xd = x.permute(0, 2, 3, 1).contiguous().cuda().bfloat16()
wd = w.permute(2, 3, 0, 1).reshape(9, 64, 64).contiguous().cuda().bfloat16()
for variant in (0, 1):
    out = torch.zeros(128, 64, device="cuda")
    rc = L.cpb200_probe_halo(xd.data_ptr(), wd.data_ptr(), out.data_ptr(), variant, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    d = (out.cpu() - ref).abs()
    bad_rows = (d.max(dim=1).values > 0).nonzero().flatten().tolist()
    print("HALO " + json.dumps({"variant": variant, "rc": rc, "max_err": float(d.max()), "bad_frac": float((d > 0).float().mean()),
                                "bad_rows": bad_rows[:40]}))
