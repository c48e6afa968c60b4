"""The compiled kernels issue their wgmma groups as built: ptxas neither injects warpgroup.arrive before a wgmma
(C7519: accumulator registers touched inside the asynchronous window) nor serialises wgmma instructions.  Reads the
per-source ptxas logs the build writes next to the objects (occdepth_b200/lib/obj/*.o.log)."""
import glob
import os

import pytest

OBJ = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "occdepth_b200", "lib", "obj")
BAD = ("C7519", "warpgroup.arrive is injected", "wgmma.mma_async instructions are serialized")


def test_no_injected_or_serialized_wgmma():
    logs = sorted(glob.glob(os.path.join(OBJ, "*.o.log")))
    if not logs:
        pytest.skip("library not built (no ptxas logs under occdepth_b200/lib/obj)")
    assert any(os.path.basename(p).startswith("conv") for p in logs)
    hits = []
    for p in logs:
        with open(p) as f:
            for line in f:
                if any(b in line for b in BAD):
                    hits.append("%s: %s" % (os.path.basename(p), line.strip()[:200]))
    assert not hits, "\n".join(hits[:20])
