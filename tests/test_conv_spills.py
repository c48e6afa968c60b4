"""Every instantiation of the tensor-core convolution kernels fits its registers: ptxas reports 0 bytes of spill
stores and loads for each of them (a ping-pong warpgroup holds a whole 128 x N accumulator tile, N registers per
thread).  Reads the per-source ptxas logs the build writes next to the objects (occdepth_b200/lib/obj/*.o.log)."""
import glob
import os
import re

import pytest

OBJ = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "occdepth_b200", "lib", "obj")
ENTRY = re.compile(r"Compiling entry function '(\w+)'")
SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")


def test_conv_kernels_do_not_spill():
    logs = sorted(glob.glob(os.path.join(OBJ, "conv*.o.log")))
    if not logs:
        pytest.skip("library not built (no ptxas logs under occdepth_b200/lib/obj)")
    kernels, bad = {}, []
    for p in logs:
        entry = None
        with open(p) as f:
            for line in f:
                m = ENTRY.search(line)
                if m:
                    entry = m.group(1)
                    continue
                m = SPILL.search(line)
                if m and entry and re.search(r"conv_(tc|halo|halox)_kernel", entry):
                    kernels[entry] = (int(m.group(1)), int(m.group(2)))
                    if kernels[entry] != (0, 0):
                        bad.append("%s: %s" % (entry, m.group(0)))
                    entry = None
    # per element type: per-tap 16 N tiles cooperative + 8 ping-pong, x-packed per-tap 5 + 2, halo 4, x-packed
    # halo 5 + 2
    assert len(kernels) == 2 * (16 + 8 + 5 + 2 + 4 + 5 + 2), sorted(kernels)
    assert not bad, "\n".join(bad)
