"""The ping-pong schedule of the tensor-core convolution kernels (N tile <= 128, at least 4 M tiles per CTA and, for
the per-tap kernel, a mainloop no shorter than the epilogue: each MMA warpgroup owns whole M tiles, alternately)
against torch on the same rounded operands, both precision modes.  The cases cover the tile-ownership and ring
bookkeeping corner cases: every ping-pong N tile, CTAs with an odd number of tiles, the tap groups of a transposed conv, the x-packed halo kernel's plane ring (CTA shares that cross a column)
and its box mode with two M tiles per box, several sources, both residual placements and both second outputs.  Each
case checks through the plan's schedule query which schedule ran; single-tile CTAs, wide tiles and store-bound 1x1
convs stay cooperative."""
import pytest

import gpu_cases as G

pytestmark = pytest.mark.gpu

PP_TILES = list(range(16, 129, 16))   # per-tap kernel widths that run ping-pong (conv_kernels.cuh: kPingPongMaxN)

CASES = {
    # per-tap, one 3x3x3 conv per ping-pong width over 640 M tiles (the widest tile == Cout wins)
    **{"tc_n%d" % n: ("tc", dict(Cin=16, Cout=n, dims=(16, 40, 128), act="leaky"), n, None) for n in PP_TILES},
    # 529 M tiles on 132 CTAs: CTA 0 takes five (warpgroup 1 three of them), the rest four
    "tc_odd_tiles": ("tc", dict(k=(1, 1, 1), Cin=128, Cout=16, dims=(1, 529, 128), res=True), 16, 529),
    "tc_planar_out1": ("tc", dict(Cin=96, Cout=20, dims=(8, 80, 128), planar=True, act="none"), 32, None),
    "tc_pre_out1_res2": ("tc", dict(Cin=64, Cout=80, dims=(8, 80, 128), pre=True, res=True, res_post=True), 80, None),
    # x-packed per-tap: N = 3 * Cout
    "tcx_n48": ("tcx", dict(k=(1, 3, 3), Cin=40, Cout=16, dims=(1, 384, 600), act="leaky"), 48, None),
    "tcx_n96": ("tcx", dict(k=(1, 3, 3), Cin=40, Cout=32, dims=(1, 384, 600), act="leaky", res=True), 96, None),
    # x-packed halo: the head's shape (TF32: plane ring; bf16: box, two M tiles per box), 40 planes x 16 H tiles
    # shared by 132 CTAs so that most shares cross a column; dilation 3 walks the residue classes as columns too
    "halox_head_d1": ("halox", dict(Cin=32, Cout=32, dims=(40, 64, 32), res=True), 96, None),
    "halox_head_d3": ("halox", dict(Cin=32, Cout=32, dims=(40, 64, 32), dil=(3, 3, 3), res=True, res_post=True),
                      96, None),
    "halox_n48_planar": ("halox", dict(Cin=32, Cout=16, dims=(40, 128, 16), planar=True, act="none"), 48, None),
    "halox_2d_n96": ("halox", dict(k=(1, 3, 3), Cin=32, Cout=32, dims=(24, 96, 32), act="leaky"), 96, None),
}
# 2 M tiles, one per CTA: cooperative, so that both warpgroups share the tile
SMALL = ("tc", dict(Cin=32, Cout=16, dims=(2, 8, 16), res=True, res_post=True), 16, 2)


def _impl(kern):
    from occdepth_b200 import _lib
    return {"tc": _lib.CONV_IMPL_TC, "tcx": _lib.CONV_IMPL_TCX, "halox": _lib.CONV_IMPL_HALOX}[kern]


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_conv_pingpong(name, precision):
    kern, kw, n_tile, n_tiles = CASES[name]
    e, info = G.conv_case(_impl(kern), precision=precision, **kw)
    assert info["schedule"] == "pingpong" and info["N_tile"] == n_tile, info
    if n_tiles is not None:
        assert info["grid_y"] == n_tiles and info["grid_x"] == min(n_tiles, 132), info
    assert e <= G.TOL[precision], (e, info)


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_conv_pingpong_halox_modes(precision):
    """the head's shape runs the plane ring in TF32 (4 single-plane stages) and the box with nM = 2 in bf16"""
    _, kw, _, _ = CASES["halox_head_d1"]
    _, info = G.conv_case(_impl("halox"), precision=precision, **kw)
    assert info["stages"] == (401 if precision == "tf32" else 302), info


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_conv_pingpong_tap_groups_and_sources(precision):
    from occdepth_b200 import _lib
    # 8 sub-pixel phases, 8..1 taps each
    e, info = G.convT_case(_lib.CONV_IMPL_TC, dims=(16, 32, 32), precision=precision)
    assert info["schedule"] == "pingpong", info
    assert e <= G.TOL[precision], (e, info)
    e, info = G.multi_case(_lib.CONV_IMPL_TC, dims=(16, 64, 80), precision=precision)   # three sources, res1
    assert info["schedule"] == "pingpong", info
    assert e <= G.TOL[precision], (e, info)


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_conv_cooperative(precision):
    """wide N tiles, CTAs with few tiles and store-bound 1x1 convs run the cooperative schedule"""
    from occdepth_b200 import _lib
    e, info = G.conv_case(_lib.CONV_IMPL_TC, precision=precision, Cin=64, Cout=160, dims=(8, 80, 128))
    assert info["N_tile"] == 160 and info["schedule"] == "cooperative", info
    assert e <= G.TOL[precision], (e, info)
    kern, kw, n_tile, n_tiles = SMALL
    e, info = G.conv_case(_impl(kern), precision=precision, **kw)
    assert info["schedule"] == "cooperative" and info["N_tile"] == n_tile and info["grid_y"] == n_tiles, info
    assert e <= G.TOL[precision], (e, info)
    e, info = G.conv_case(_lib.CONV_IMPL_TC, precision=precision, k=(1, 1, 1), Cin=32, Cout=64, dims=(1, 330, 512))
    assert info["schedule"] == "cooperative", info
    assert e <= G.TOL[precision], (e, info)
