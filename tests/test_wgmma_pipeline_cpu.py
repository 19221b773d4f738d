"""CPU test (-m "not gpu"): every wgmma kernel of the built library keeps its tensor-core instructions pipelined.

When ptxas cannot keep several wgmma.mma_async in flight it does not fail: it prints an "info" line (C7511, "wgmma
instructions are serialized") and waits for every HGMMA to finish before the next one issues.  The kernels still
compute the same results, so only a GPU run shows it (the DLA-34 fp16x2 headline loses about 8 %).  A known trigger is
two in-flight wgmma whose accumulator register lists partly overlap, e.g. an m64n(2N)k16 into [acc | acc2] followed by
an m64nNk16 into acc2 alone.

In the SASS a serialised kernel is recognisable without a GPU: each HGMMA is followed by a full drain
(WARPGROUP.DEPBAR.LE gsb0, 0x0) before the next HGMMA.  A pipelined kernel drains once or twice per tile, at the end
of its K loop or before its epilogue."""
import os
import re
import shutil
import subprocess

import pytest


def drained_hgmma(sass):
    """{function: (HGMMA count, HGMMAs followed by a full wgmma drain before the next HGMMA)} of cuobjdump -sass text."""
    out, fn, pending = {}, None, False
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn, pending = m.group(1), False
            continue
        if fn is None:
            continue
        if "HGMMA" in line:
            t, d = out.get(fn, (0, 0))
            out[fn] = (t + 1, d)
            pending = True
        elif pending and re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0\b", line):
            t, d = out[fn]
            out[fn] = (t, d + 1)
            pending = False
    return out


def serialized_kernels(libpath):
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([tool, "-sass", libpath], capture_output=True, text=True, check=True).stdout
    counts = drained_hgmma(sass)
    assert counts, "no wgmma kernels found in the library"
    return sorted(f"{fn}: {d} of {t} HGMMA drained" for fn, (t, d) in counts.items() if t > 2 and 2 * d > t)


def test_drain_detector_on_constructed_sass():
    pipelined = """
        Function : _Z1kv
        /*0100*/ WARPGROUP.ARRIVE ;
        /*0110*/ HGMMA.64x64x16.F32 R24, gdesc[UR8], R24, gsb0 ;
        /*0120*/ WARPGROUP.ARRIVE ;
        /*0130*/ HGMMA.64x64x16.F32 R56, gdesc[UR8], R56, gsb0 ;
        /*0140*/ WARPGROUP.DEPBAR.LE gsb0, 0x1 ;
        /*0150*/ HGMMA.64x64x16.F32 R24, gdesc[UR8], R24, gsb0 ;
        /*0160*/ WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
    """
    serial = """
        Function : _Z1sv
        /*0100*/ HGMMA.64x128x16.F32 R24, gdesc[UR8], R24, gsb0 ;
        /*0110*/ WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        /*0120*/ WARPGROUP.ARRIVE ;
        /*0130*/ HGMMA.64x64x16.F32 R56, gdesc[UR8], R56, gsb0 ;
        /*0140*/ WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        /*0150*/ WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
    """
    assert drained_hgmma(pipelined + serial) == {"_Z1kv": (3, 1), "_Z1sv": (2, 2)}


def test_no_wgmma_kernel_is_serialized():
    from centerpose_b200 import _lib
    if not os.path.exists(_lib.LIBPATH):
        pytest.skip("the CUDA library has not been built")
    bad = serialized_kernels(_lib.LIBPATH)
    assert not bad, "wgmma kernels that wait for every HGMMA (ptxas C7511):\n" + "\n".join(bad)
