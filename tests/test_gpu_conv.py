"""Implicit-GEMM convolution through the C ABI: wgmma paths and the SIMT path vs torch fp32 on operands rounded
to the mode's element type (TF32 values in fp32 containers / bf16), both precision modes."""
import pytest

import gpu_cases as G

pytestmark = pytest.mark.gpu
PREC = pytest.mark.parametrize("precision", G.PRECISIONS)


@PREC
@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case", sorted(G.CONV_CASES))
def test_conv(impl, case, precision):
    from occdepth_b200 import _lib
    e, info = G.conv_case(_lib.CONV_IMPL_TC if impl == "tc" else _lib.CONV_IMPL_SIMT, precision=precision,
                          **G.CONV_CASES[case])
    assert e <= G.TOL[precision], (e, info)


@PREC
@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_conv_transpose_and_multi(impl, precision):
    from occdepth_b200 import _lib
    i = _lib.CONV_IMPL_TC if impl == "tc" else _lib.CONV_IMPL_SIMT
    e, info = G.convT_case(i, precision=precision)
    assert e <= G.TOL[precision], (e, info)
    e, info = G.multi_case(i, precision=precision)
    assert e <= G.TOL[precision], (e, info)


@PREC
def test_conv_transpose_grouped_launch(precision, monkeypatch):
    """the 8 sub-pixel phases as tap groups of ONE launch (default) == the 8 separate launches, bit for bit; the
    level shapes of the 3-D decoder (odd extents, Cout 32 / 64)"""
    import torch
    from occdepth_b200.engine import CL, Plan
    dev = torch.device("cuda")
    for (ci, co, dims) in ((32, 16, (4, 6, 5)), (64, 32, (9, 7, 16)), (128, 64, (5, 8, 4))):
        g = torch.Generator().manual_seed(3)
        x = G.rnd(precision)(torch.randn(1, ci, *dims, generator=g)).to(dev)
        w = G.rnd(precision)(torch.randn(ci, co, 3, 3, 3, generator=g) / (ci * 8) ** 0.5).to(dev)
        b = torch.randn(co, generator=g).to(dev)
        sk = G.rnd(precision)(torch.randn(1, co, *[2 * d for d in dims], generator=g)).to(dev)
        outs, n_ops = [], []
        for grouped in ("1", "0"):
            monkeypatch.setenv("OCCDEPTH_CONVT_GROUPED", grouped)
            plan = Plan(dev, precision=precision)
            y = plan.conv_transpose_k3s2(CL.from_planar(x, precision=precision), w, b, act="relu",
                                         res_post=CL.from_planar(sk, precision=precision))
            plan.run()
            torch.cuda.synchronize()
            outs.append(y.to_planar())
            n_ops.append(len(plan.ops))
        assert n_ops == [1, 8]
        assert torch.equal(outs[0], outs[1])
        ref = torch.relu(torch.nn.functional.conv_transpose3d(x.cpu(), w.cpu(), b.cpu(), 2, 1, 1)) + sk.cpu()
        assert G.rel_err(outs[0].cpu(), ref) <= G.TOL[precision]


@PREC
def test_conv_large_vs_simt(precision):
    """full-size head conv shape (Cin=Cout=32, dil 3) on a 64x64x32 slab: auto (halo) / TC vs SIMT on the same
    buffers."""
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200.engine import CL, Plan
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(1)
    x = CL.from_planar(torch.randn(1, 32, 64, 64, 32, generator=g).cuda(), precision=precision)
    w = (torch.randn(32, 32, 3, 3, 3, generator=g) / 30).cuda()
    b = torch.randn(32, generator=g).cuda()
    outs = []
    for impl in (None, _lib.CONV_IMPL_TC, _lib.CONV_IMPL_SIMT):
        plan = Plan(dev, precision=precision)
        outs.append(plan.conv(x, w, b, padding=3, dilation=3, act="relu", impl=impl))
        plan.run()
    torch.cuda.synchronize()
    c = outs[2].buf.float()
    for o in outs[:2]:
        assert float((o.buf.float() - c).abs().max()) <= G.TOL[precision] * float(c.abs().max())


@PREC
@pytest.mark.parametrize("case", sorted(G.HALO_CASES))
def test_conv_halo(case, precision):
    """halo-tile wgmma kernel (row-shifted swizzled smem views, sub-sampled TMA for dilation)"""
    from occdepth_b200 import _lib
    kw = G.HALO_CASES[case]
    one_chunk = 32 if precision == "tf32" else 64           # the resident-weight scheme holds ONE K chunk
    if kw.get("Cin", 32) > one_chunk or (precision == "tf32" and case == "h_big"):
        # (tf32: 27 resident taps x 32 x 128 B leave no room for a W = 32 box -- auto mode uses the x-packed kernel)
        with pytest.raises(RuntimeError, match="halo"):
            G.conv_case(_lib.CONV_IMPL_HALO, precision=precision, **kw)
        return
    e, info = G.conv_case(_lib.CONV_IMPL_HALO, precision=precision, **kw)
    assert e <= G.TOL[precision], (e, info)


HALOX_CASES = {
    "hx_w32_d1": dict(Cin=32, Cout=32, dims=(6, 10, 32)),
    "hx_w32_d2_res": dict(Cin=32, Cout=32, dims=(9, 11, 32), dil=(2, 2, 2), res=True),
    "hx_w32_d3": dict(Cin=32, Cout=32, dims=(8, 13, 32), dil=(3, 3, 3)),
    "hx_w16_c16": dict(Cin=16, Cout=16, dims=(5, 9, 16)),
    "hx_w8_b2": dict(B=2, Cin=24, Cout=40, dims=(7, 6, 8), act="leaky"),
    "hx_w32_n2_planar": dict(Cin=32, Cout=2, dims=(6, 10, 32), act="none", planar=True),
    "hx_w32_n20_pre": dict(Cin=32, Cout=20, dims=(5, 12, 32), pre=True),
    "hx_2d_hw": dict(k=(1, 3, 3), Cin=32, Cout=32, dims=(1, 21, 32), act="leaky"),
    "hx_1d_w": dict(k=(1, 1, 3), Cin=16, Cout=16, dims=(6, 7, 16), dil=(1, 1, 2)),
    "hx_c8": dict(Cin=2, Cout=20, dims=(4, 9, 32), act="none"),
    "hx_big": dict(Cin=32, Cout=32, dims=(20, 40, 32)),
    "hx_big_d3_respost": dict(Cin=32, Cout=32, dims=(20, 40, 32), dil=(3, 3, 3), res=True, res_post=True),
}


@PREC
@pytest.mark.parametrize("case", sorted(HALOX_CASES))
def test_conv_halo_xpacked(case, precision):
    """x-packed halo kernel (W == one warp row: three W taps per MMA, masked lane shifts == zero padding)"""
    from occdepth_b200 import _lib
    e, info = G.conv_case(_lib.CONV_IMPL_HALOX, precision=precision, **HALOX_CASES[case])
    assert e <= G.TOL[precision], (e, info)


TCX_CASES = {
    "x_2d_multi": dict(k=(1, 3, 3), Cin=40, Cout=48, dims=(1, 13, 70), B=2),
    "x_3d_c16": dict(Cin=16, Cout=16, dims=(5, 7, 33)),
    "x_1d_w_c64": dict(k=(1, 1, 3), Cin=64, Cout=80, dims=(3, 4, 61), act="leaky"),
    "x_stride_hd": dict(Cin=24, Cout=32, dims=(6, 9, 31), stride=(2, 2, 1), res=False),
    "x_big_2d": dict(k=(1, 3, 3), Cin=80, Cout=80, dims=(1, 90, 200), res=True),
}


@PREC
@pytest.mark.parametrize("case", sorted(TCX_CASES))
def test_conv_tc_xpacked(case, precision):
    """x-packed per-tap kernel (TCX: three W taps per MMA, lane-shifted epilogue sum)"""
    from occdepth_b200 import _lib
    e, info = G.conv_case(_lib.CONV_IMPL_TCX, precision=precision, **TCX_CASES[case])
    assert e <= G.TOL[precision], (e, info)


def test_auto_picks_tcx_and_halo():
    """the default ('auto') selection: decoder-width 3x3 convs run x-packed (per-tap kernel), head convs on the
    x-packed halo kernel (W = 32 = one warp row), narrow 2-D convs on the halo kernel"""
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200.engine import Plan
    dev = torch.device("cuda")
    plan = Plan(dev)
    x = plan.alloc(1, 1, 40, 64, 80)
    plan.conv(x, torch.randn(80, 80, 1, 3, 3, device=dev), torch.zeros(80, device=dev), padding=(0, 1, 1))
    y = plan.alloc(1, 8, 16, 32, 32)
    plan.conv(y, torch.randn(32, 32, 3, 3, 3, device=dev), torch.zeros(32, device=dev), padding=1)
    z = plan.alloc(1, 1, 24, 40, 32)
    plan.conv(z, torch.randn(32, 32, 1, 3, 3, device=dev), torch.zeros(32, device=dev), padding=(0, 1, 1))
    assert plan.ops[0].impl == _lib.CONV_IMPL_TCX and plan.ops[1].impl == _lib.CONV_IMPL_HALOX
    assert plan.ops[2].impl == _lib.CONV_IMPL_HALO
