"""The x-packed epilogue's W-neighbour sums (conv_halox_kernel), one launch replayed against its float64 evaluation
with the bound of tests/conv_replay.py: dilations 1, 2 and 3 on every innermost extent a halox plan accepts (W = 32,
16, 8), in both schedules and both precisions.  Together they take the neighbour from inside a warp's 16 rows, from the
previous and next warp through the exchange buffer, and from the zero padding at the line edges.  Cout = 20 (< the
padded 32 columns) covers the channel tail with the planar fp32 output and with the class map."""
import pytest
import torch

import conv_replay as R

pytestmark = pytest.mark.gpu

# (D, H): enough M tiles for at least 4 per CTA (ping-pong), or a handful of tiles (cooperative)
GRIDS = {"pingpong": (40, 256), "cooperative": (2, 8)}


def _replay(precision, dims, d, Cout, out1_mode, schedule):
    from occdepth_b200 import _lib
    from occdepth_b200.engine import CL, ConvOp, Plan
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(d)
    plan = Plan(dev, precision=precision)
    x = plan.alloc(1, *dims, 32)
    w = (torch.randn(Cout, 32, 3, 3, 3, generator=g) / 30).to(dev)
    b = torch.randn(Cout, generator=g).to(dev)
    if out1_mode == "none":
        plan.conv(x, w, b, padding=d, dilation=d, act="relu", res1=plan.alloc(1, *dims, Cout), impl=_lib.CONV_IMPL_HALOX)
    elif out1_mode == "planar":
        out1 = torch.empty(1, Cout, *dims, device=dev)
        plan.conv(x, w, b, padding=d, dilation=d, out1=out1, out1_mode="planar", no_out0=True,
                  impl=_lib.CONV_IMPL_HALOX)
    else:
        out1 = torch.empty(*((1,) + dims), dtype=torch.uint16, device=dev)
        plan.conv(x, w, b, padding=d, dilation=d, out1=out1, out1_mode="classes", no_out0=True,
                  impl=_lib.CONV_IMPL_HALOX)
    (op,) = plan.ops
    assert isinstance(op, ConvOp) and isinstance(x, CL)
    info = op.info()
    assert info["schedule"] == schedule and info["N_tile"] == 96, info
    R.fill(op, R.seed_of(R.signature(op)))
    snap = R.Snapshot(op)
    op.run(_lib.stream_ptr())
    torch.cuda.synchronize()
    fails, _ = R.check_op(op, snap, R.reference(snap), info)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("schedule", sorted(GRIDS))
@pytest.mark.parametrize("W", (32, 16, 8))
@pytest.mark.parametrize("d", (1, 2, 3))
def test_xp_neighbours(d, W, schedule, precision):
    _replay(precision, GRIDS[schedule] + (W,), d, 32, "none", schedule)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("schedule", sorted(GRIDS))
@pytest.mark.parametrize("out1_mode", ("planar", "classes"))
def test_xp_channel_tail(out1_mode, schedule, precision):
    _replay(precision, GRIDS[schedule] + (16,), 2, 20, out1_mode, schedule)
