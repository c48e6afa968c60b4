"""UpSampleBN's conv1 split into a coarse per-tap GEMM, a resize-and-sum of its nine products and the skip-half conv
(occdepth_b200/models/unet2d.py): the identity, restated in float64 with F.interpolate / F.conv2d, must equal
conv3x3(cat(interpolate(x), skip)) to rounding, for the packing order of pack_tap_weights."""
import contextlib
import io

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F


def tapsum_ref(Y, co, tap_stride, OH, OW):
    """S[b, c, p] = sum_t [p+t inside OH x OW] bilinear_ac(Y_t)(p+t)[c], Y_t = Y[:, t*tap_stride : t*tap_stride+co]"""
    S = 0
    for t in range(9):
        dy, dx = t // 3 - 1, t % 3 - 1
        U = F.interpolate(Y[:, t * tap_stride:t * tap_stride + co], size=(OH, OW), mode="bilinear", align_corners=True)
        Up = F.pad(U, (1, 1, 1, 1))                   # the fine grid's zero padding = the in-bounds mask
        S = S + Up[:, :, 1 + dy:1 + dy + OH, 1 + dx:1 + dx + OW]
    return S


def _block(c_up, c_skip, co, seed):
    from occdepth_b200.models.unet2d import UpSampleBN
    torch.manual_seed(seed)
    m = UpSampleBN(c_up + c_skip, co).eval()
    for bn in (m._net[1], m._net[4]):
        bn.running_mean.uniform_(-0.5, 0.5)
        bn.running_var.uniform_(0.5, 2.0)
        bn.weight.data.uniform_(0.5, 1.5)
        bn.bias.data.uniform_(-0.5, 0.5)
    return m


def split_conv1(m, x, skip):
    """float64 restatement of what UpSampleBN.emit plans: pre-activation of conv1 + BN"""
    from occdepth_b200.engine import fold_bn
    from occdepth_b200.models.unet2d import pack_tap_weights
    w1, b1 = fold_bn(m._net[0].weight, m._net[0].bias, m._net[1])
    w1, b1 = w1.double(), b1.double()
    c_up, co = x.shape[1], w1.shape[0]
    wy = pack_tap_weights(w1[:, :c_up])
    Y = torch.einsum("kc,bchw->bkhw", wy, x)          # the coarse 1x1 GEMM
    S = tapsum_ref(Y, co, wy.shape[0] // 9, skip.shape[2], skip.shape[3])
    P = F.conv2d(skip, w1[:, c_up:], b1, padding=1)  # the skip half, bias included
    want = F.conv2d(torch.cat([F.interpolate(x, size=skip.shape[2:], mode="bilinear", align_corners=True), skip], 1),
                    w1, b1, padding=1)
    return P + S, want


def test_pack_tap_weights_order():
    from occdepth_b200.models.unet2d import pack_tap_weights
    w = torch.randn(12, 5, 3, 3, dtype=torch.float64)
    wy = pack_tap_weights(w)
    assert tuple(wy.shape) == (9 * 16, 5)             # 12 output channels -> tap blocks of 16 (vector aligned)
    for t in range(9):
        dy, dx = t // 3 - 1, t % 3 - 1
        assert torch.equal(wy[t * 16:t * 16 + 12], w[:, :, dy + 1, dx + 1])
        assert not wy[t * 16 + 12:(t + 1) * 16].any()


# B7 decoder levels (coarse -> fine of the benchmark frame) at reduced widths, and degenerate extents where the
# align_corners scale is 0 (one coarse or one fine row / column)
@pytest.mark.parametrize("hw,OHW", [((14, 45), (24, 86)), ((24, 86), (47, 172)), ((47, 172), (94, 343)),
                                    ((1, 5), (3, 9)), ((4, 1), (7, 3)), ((3, 4), (1, 6)), ((5, 3), (9, 1)),
                                    ((1, 1), (4, 4)), ((6, 7), (6, 7))])
@pytest.mark.parametrize("co", [8, 12])
def test_split_equals_conv_of_concat(hw, OHW, co):
    m = _block(16, 8, co, seed=hw[0] * 31 + OHW[1])
    g = torch.Generator().manual_seed(co + hw[1])
    x = torch.randn(2, 16, *hw, generator=g, dtype=torch.float64)
    skip = torch.randn(2, 8, *OHW, generator=g, dtype=torch.float64)
    with torch.no_grad():
        got, want = split_conv1(m, x, skip)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_split_on_the_bias_bordered_map():
    """up16 reads dec.conv2's output: a 1x1 conv with padding=1, so its one-pixel border is the bias alone"""
    m = _block(24, 8, 16, seed=3)
    g = torch.Generator().manual_seed(1)
    bias = torch.randn(24, 1, 1, generator=g, dtype=torch.float64)
    x = bias.expand(24, 14, 45).clone()
    x[:, 1:-1, 1:-1] += torch.randn(24, 12, 43, generator=g, dtype=torch.float64)
    x = torch.stack([x, x.flip(2)])
    skip = torch.randn(2, 8, 24, 86, generator=g, dtype=torch.float64)
    with torch.no_grad():
        got, want = split_conv1(m, x, skip)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def test_decoder_plan_forms_and_reference_flops(monkeypatch):
    """the planned B7 decoder: the wide levels (Cout 1280 / 640 / 320) run coarse GEMM + skip conv + tap sum without
    a resize launch, the narrow ones (160 / 80) resize + two-source conv; the FLOP bookkeeping of the split levels still
    adds up to the reference convolutions' 2*MACs"""
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")           # host-only plan build
    from occdepth_b200.engine import Plan
    from occdepth_b200.models.unet2d import UNet2D, split_pays
    with contextlib.redirect_stdout(io.StringIO()):
        m = UNet2D.build(out_feature=64, use_decoder=True, backbone_2d_name="tf_efficientnet_b7_ns",
                         return_up_feats=1).eval()
    plan = Plan(torch.device("cpu"))
    x = plan.alloc(1, 1, 376, 1370, 3)
    with torch.no_grad():
        m.emit(plan, x)
    dec = m.decoder
    sizes = {16: ((14, 45), (24, 86)), 8: ((24, 86), (47, 172)), 4: ((47, 172), (94, 343)),
             2: ((94, 343), (188, 685)), 1: ((188, 685), (376, 1370))}
    assert [split_pays(getattr(dec, "up%d" % s)._net[0].weight.shape[0]) for s in sizes] == [True] * 3 + [False] * 2
    for s, ((h, w), (OH, OW)) in sizes.items():
        up = getattr(dec, "up%d" % s)
        co, cin = up._net[0].weight.shape[:2]
        ops = {op.name: op for op in plan.ops if op.name.startswith("up%d." % s)}
        if not split_pays(co):
            assert set(ops) == {"up%d.%s" % (s, k) for k in ("bilinear", "conv1", "conv2")}, sorted(ops)
            assert ops["up%d.conv1" % s].flops == 2 * OH * OW * co * 9 * cin
            continue
        assert set(ops) == {"up%d.%s" % (s, k) for k in ("taps", "conv1", "tapsum", "conv2")}, sorted(ops)
        c_skip = ops["up%d.conv1" % s].flops // (2 * OH * OW * co * 9)
        c_up = cin - c_skip
        assert ops["up%d.taps" % s].flops == 2 * h * w * 9 * co * c_up                  # executed
        assert ops["up%d.taps" % s].flops + ops["up%d.tapsum" % s].flops == 2 * OH * OW * co * 9 * c_up  # reference
        assert ops["up%d.taps" % s].flops < ops["up%d.tapsum" % s].flops
