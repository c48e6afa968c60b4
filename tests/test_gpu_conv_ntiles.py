"""Every compiled N tile of every tensor-core convolution kernel, both precision modes, against the SIMT kernel on the
same buffers.  The kernels are compiled once per N tile; the shapes below are chosen so that the planner selects each
width, and the last test checks that together they cover exactly the compiled menu."""
import pytest

import gpu_cases as G

pytestmark = pytest.mark.gpu

# compiled N tiles per kernel (conv_kernels.cuh: TcTiles, TcxTiles, HaloxTiles, HaloTiles)
MENU = {
    "tc": set(range(16, 257, 16)),
    "tcx": {48, 96, 144, 192, 240},
    "halox": {48, 96, 144, 192, 240},
    "halo": {16, 32, 48, 64},
}

# kernel -> list of (Cout, conv kwargs).  Per-tap: a 1x1 conv with Cout = N over 1320 M tiles (10 waves of 132 CTAs
# at N = Cout), where every divisor of Cout costs the same number of epilogue waves and the widest tile wins.
CASES = {
    "tc": [(n, dict(k=(1, 1, 1), dims=(1, 330, 512), Cin=32)) for n in sorted(MENU["tc"])],
    "tcx": [(n // 3, dict(k=(1, 3, 3), dims=(1, 24, 70), Cin=40)) for n in sorted(MENU["tcx"])],
    "halox": [(n // 3, dict(k=(1, 3, 3), dims=(2, 12, 32), Cin=32)) for n in sorted(MENU["halox"])],
    "halo": [(n, dict(k=(1, 3, 3), dims=(1, 21, 40), Cin=32)) for n in sorted(MENU["halo"])],
}
IDS = [(kern, i) for kern in CASES for i in range(len(CASES[kern]))]
_seen = {}


def _run(kern, Cout, k, dims, Cin, precision):
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200.engine import CL, Plan
    impl = {"tc": _lib.CONV_IMPL_TC, "tcx": _lib.CONV_IMPL_TCX, "halox": _lib.CONV_IMPL_HALOX,
            "halo": _lib.CONV_IMPL_HALO}[kern]
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(Cout)
    x = CL.from_planar(torch.randn(1, Cin, *dims, generator=g).to(dev), precision=precision)
    w = (torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5).to(dev)
    b = torch.randn(Cout, generator=g).to(dev)
    pad = tuple((kk - 1) // 2 for kk in k)
    outs, infos = [], []
    for i in (impl, _lib.CONV_IMPL_SIMT):
        plan = Plan(dev, precision=precision)
        outs.append(plan.conv(x, w, b, padding=pad, act="leaky", impl=i))
        infos.append(plan.ops[0].info())
        plan.run()
    torch.cuda.synchronize()
    got, want = outs[0].buf.float(), outs[1].buf.float()
    return float((got - want).abs().max() / want.abs().max()), infos[0]


# both outputs are rounded to the storage type, each within G.TOL of the exact result: they differ by up to twice that
def _tol(precision):
    return 2 * G.TOL[precision]


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("kern,idx", IDS, ids=["%s-%d" % (k, i) for k, i in IDS])
def test_conv_ntile(kern, idx, precision):
    Cout, kw = CASES[kern][idx]
    e, info = _run(kern, Cout, precision=precision, **kw)
    _seen.setdefault((kern, precision), set()).add(info["N_tile"])
    assert e <= _tol(precision), (e, info)


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_conv_ntile_menu_covered(precision):
    """the cases above ran every compiled N tile of every kernel, and nothing else"""
    for kern in CASES:
        seen = _seen.get((kern, precision))
        if seen is None or len(seen) < len(CASES[kern]):   # run on its own: plan (and run) the cases here
            seen = {_run(kern, Cout, precision=precision, **kw)[1]["N_tile"] for Cout, kw in CASES[kern]}
        assert seen == MENU[kern], (kern, precision, sorted(seen))
