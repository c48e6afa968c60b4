"""UpSampleBN with the resize behind conv1's taps on the GPU: occd_upsample_tapsum_ac against its float64
restatement, one planned block at the real B7 up16 / up4 shapes against torch fp32 conv(cat(interpolate)), and which
levels of a planned decoder run split."""
import contextlib
import io

import pytest
import torch
import torch.nn.functional as F

import gpu_cases as G
from test_upconv_split_host import _block, tapsum_ref

pytestmark = pytest.mark.gpu
PREC = pytest.mark.parametrize("precision", G.PRECISIONS)
TDT = {"tf32": torch.float32, "bf16": torch.bfloat16}
SENTINEL = -448.0          # exact in bf16 and TF32: channels the kernel must not touch keep it


def L():
    from occdepth_b200 import _lib
    return _lib.lib()


def st():
    from occdepth_b200 import _lib
    return _lib.stream_ptr()


def code(precision):
    return 0 if precision == "tf32" else 1


def _launch(y, pre, out, precision, B, h, w, OH, OW, C_, cs_y, y_off, ts, cs_pre, pre_off, cs_out, out_off, act):
    return L().occd_upsample_tapsum_ac(y.data_ptr(), pre.data_ptr() if pre is not None else None, out.data_ptr(),
                                       code(precision), B, h, w, OH, OW, C_, cs_y, y_off, ts, cs_pre, pre_off, cs_out,
                                       out_off, act, st())


@PREC
@pytest.mark.parametrize("h,w,OH,OW", [(7, 9, 12, 22), (14, 45, 24, 86), (1, 5, 3, 9), (6, 1, 11, 3), (5, 6, 1, 1),
                                       (9, 13, 1, 20), (4, 4, 4, 4), (33, 70, 65, 139)])
@pytest.mark.parametrize("with_pre", [False, True])
def test_tapsum_kernel(precision, h, w, OH, OW, with_pre):
    """channel windows: Y's taps at y_off + t*ts inside a wider row, pre and out sharing one buffer window (in place)"""
    from occdepth_b200 import _lib
    g = torch.Generator().manual_seed(h * 1000 + OW)
    tdt, rnd = TDT[precision], G.rnd(precision)
    B, C_, ts, y_off, cs_y = 2, 24, 32, 8, 8 + 9 * 32 + 16
    cs_out, out_off = 48, 16
    Y = rnd(torch.randn(B, 9 * ts, h, w, generator=g))
    yin = torch.full((B, h, w, cs_y), float("nan"), dtype=tdt)
    yin[..., y_off:y_off + 9 * ts] = Y.permute(0, 2, 3, 1).to(tdt)
    want = tapsum_ref(Y.double(), C_, ts, OH, OW)
    buf = torch.full((B, OH, OW, cs_out), SENTINEL, dtype=tdt)
    act = _lib.ACT_NONE
    if with_pre:
        pre = rnd(torch.randn(B, C_, OH, OW, generator=g))
        buf[..., out_off:out_off + C_] = pre.permute(0, 2, 3, 1).to(tdt)
        want = F.leaky_relu(want + pre.double(), 0.01)
        act = _lib.ACT_LEAKY
    out = buf.cuda()
    yc = yin.cuda()
    assert _launch(yc, out if with_pre else None, out, precision, B, h, w, OH, OW, C_, cs_y, y_off, ts, cs_out,
                   out_off, cs_out, out_off, act) == 0
    torch.cuda.synchronize()
    oc = out.float().cpu()
    assert torch.all(oc[..., :out_off] == SENTINEL) and torch.all(oc[..., out_off + C_:] == SENTINEL)
    got = oc[..., out_off:out_off + C_].permute(0, 3, 1, 2)
    if precision == "tf32":
        assert torch.equal(got, G.tf32r(got))
    err = G.rel_err(got.double(), want)
    G.record("tapsum.%dx%d_%dx%d.%s" % (h, w, OH, OW, "pre" if with_pre else "sum"), precision, rel=err)
    assert err <= G.TOL[precision], err


def test_tapsum_refuses_bad_arguments():
    y = torch.zeros(1, 4, 4, 9 * 16, device="cuda")
    out = torch.zeros(1, 8, 8, 16, device="cuda")
    ok = dict(B=1, h=4, w=4, OH=8, OW=8, C_=16, cs_y=144, y_off=0, ts=16, cs_pre=16, pre_off=0, cs_out=16, out_off=0,
              act=0)

    def call(**kw):
        a = dict(ok, **kw)
        return _launch(y, None, out, "tf32", a["B"], a["h"], a["w"], a["OH"], a["OW"], a["C_"], a["cs_y"], a["y_off"],
                       a["ts"], a["cs_pre"], a["pre_off"], a["cs_out"], a["out_off"], a["act"])

    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(h=0), dict(OW=0), dict(C_=0), dict(ts=12), dict(ts=8), dict(cs_y=136), dict(y_off=8),
                dict(cs_out=12), dict(out_off=8), dict(C_=24), dict(act=9), dict(B=70000)):
        assert call(**bad) != 0, bad
    assert L().occd_upsample_tapsum_ac(None, None, out.data_ptr(), 0, 1, 4, 4, 8, 8, 16, 144, 0, 16, 16, 0, 16, 0, 0,
                                       st()) != 0
    assert L().occd_upsample_tapsum_ac(y.data_ptr(), None, out.data_ptr(), 5, 1, 4, 4, 8, 8, 16, 144, 0, 16, 16, 0,
                                       16, 0, 0, st()) != 0


# the real B7 levels of the benchmark frame: (C_up, C_skip, Cout, coarse, fine)
LEVELS = {"up16": (2560, 224, 1280, (14, 45), (24, 86)), "up4": (640, 48, 320, (47, 172), (94, 343))}
# about 2x the figures measured on an H100 (tf32 4.6e-4, bf16 4.5e-3)
BLOCK_TOL = {"tf32": 1e-3, "bf16": 1e-2}


@PREC
@pytest.mark.parametrize("level", sorted(LEVELS))
def test_upsample_block_real_shapes(precision, level):
    from occdepth_b200.engine import CL, Plan
    c_up, c_skip, co, hw, OHW = LEVELS[level]
    m = _block(c_up, c_skip, co, seed=7)
    g = torch.Generator().manual_seed(11)
    rnd = G.rnd(precision)
    x = rnd(torch.randn(1, c_up, *hw, generator=g)).cuda()
    skip = rnd(torch.randn(1, c_skip, *OHW, generator=g)).cuda()
    m = m.cuda()
    tf = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            want = m._net(torch.cat([F.interpolate(x, size=OHW, mode="bilinear", align_corners=True), skip], 1))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf
    plan = Plan(torch.device("cuda"), precision=precision)
    with torch.no_grad():
        y = m.emit(plan, CL.from_planar(x, precision=precision), CL.from_planar(skip, precision=precision), level)
    assert [op.name.split(".")[1] for op in plan.ops] == ["taps", "conv1", "tapsum", "conv2"]
    plan.run()
    torch.cuda.synchronize()
    err = G.rel_err(y.to_planar(squeeze_d=True).double(), want.double())
    G.record("upsample_block.%s" % level, precision, rel=err)
    assert err <= BLOCK_TOL[precision], err


@PREC
def test_planned_decoder_forms(precision):
    """B3 decoder widths 768 / 384 / 192 / 96 / 48: three split levels (no resize launch), two narrow ones resized"""
    from occdepth_b200.models.unet2d import UNet2D
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = UNet2D.build(out_feature=32, use_decoder=True, backbone_2d_name="tf_efficientnet_b3_ns",
                         return_up_feats=1).eval()
    m = m.cuda().set_precision(precision)
    with torch.no_grad():
        out = m(torch.randn(1, 3, 38, 45, device="cuda"))
    assert all(torch.isfinite(v).all() for v in out.values())
    ops = [op for plan, *_ in m._plans().values() for op in plan.ops]
    names = [getattr(op, "name", "") for op in ops]
    assert [n.split(".")[0] for n in names if n.endswith(".tapsum")] == ["up16", "up8", "up4"]
    assert [n.split(".")[0] for n in names if n.endswith(".bilinear")] == ["up2", "up1"]
