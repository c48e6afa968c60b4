"""tf_efficientnet_b{3,4,5,7}_ns with geffnet's module names (what the reference's torch.hub.load returns at
occdepth/models/unet2d.py:238-240), as a parameter holder + sm_90a launch emitter.

State-dict keys equal geffnet's (`conv_stem, bn1, blocks.S.B.{conv_pw,bn1,conv_dw,bn2,se.conv_reduce,
se.conv_expand,conv_pwl,bn3}, conv_head, bn2, classifier`), so reference checkpoints
(`net_rgb.encoder.original_model.*`) load with strict=True.  Architecture per the published EfficientNet
definition: see `block_specs`.  TF "SAME" padding, Swish, BN eps 1e-3.
"""
import math
import os

import torch
import torch.nn as nn

from .. import _lib
from ..engine import ConvOp, FnOp, fold_bn, _round_up

ARCH = [("ds", 1, 3, 1, 1, 16), ("ir", 2, 3, 2, 6, 24), ("ir", 2, 5, 2, 6, 40), ("ir", 3, 3, 2, 6, 80),
        ("ir", 3, 5, 1, 6, 112), ("ir", 4, 5, 2, 6, 192), ("ir", 1, 3, 1, 6, 320)]
MULTS = {"tf_efficientnet_b3_ns": (1.2, 1.4), "tf_efficientnet_b4_ns": (1.4, 1.8),
         "tf_efficientnet_b5_ns": (1.6, 2.2), "tf_efficientnet_b7_ns": (2.0, 3.1)}
BN_EPS = 1e-3


def _round_channels(c, mult, divisor=8):
    c = c * mult
    n = max(divisor, int(c + divisor / 2) // divisor * divisor)
    return n + divisor if n < 0.9 * c else n


def block_specs(name):
    wm, dm = MULTS[name]
    stem = _round_channels(32, wm)
    specs, cin = [], stem
    for si, (typ, r, k, s, e, c) in enumerate(ARCH):
        cout = _round_channels(c, wm)
        for bi in range(int(math.ceil(r * dm))):
            specs.append((si, typ, cin, cout, k, s if bi == 0 else 1, e, max(1, int(cin * 0.25 + 0.5))))
            cin = cout
    return stem, specs, _round_channels(1280, wm)


def same_pad(i, k, s):
    """TF SAME: total padding so that out = ceil(i / s); the odd pixel goes to the bottom/right."""
    return max((math.ceil(i / s) - 1) * s + (k - 1) + 1 - i, 0)


def _conv(cin, cout, k, stride=1, groups=1, bias=False):
    # parameter holder only (the TF-SAME geometry is applied by the emitter)
    return nn.Conv2d(cin, cout, k, stride, 0 if stride > 1 else (k - 1) // 2, groups=groups, bias=bias)


class SqueezeExcite(nn.Module):
    def __init__(self, chs, reduce_chs):
        super().__init__()
        self.conv_reduce = nn.Conv2d(chs, reduce_chs, 1, bias=True)
        self.act1 = nn.SiLU()
        self.conv_expand = nn.Conv2d(reduce_chs, chs, 1, bias=True)


def _dw_entry(L):
    """depthwise entry point: the shared-memory-tiled kernel by default; OCCDEPTH_DW_IMPL=direct selects the
    register-window variant."""
    impl = os.environ.get("OCCDEPTH_DW_IMPL", "tiled")
    if impl not in ("tiled", "direct"):
        raise ValueError(f"OCCDEPTH_DW_IMPL must be 'tiled' or 'direct', got {impl!r}")
    return L.occd_dwconv2d_tiled_fwd if impl == "tiled" else L.occd_dwconv2d_fwd


def _emit_dw_se_project(plan, x, conv_dw, bn_dw, se, conv_proj, bn_proj, k, stride, residual, out=None, name=""):
    """dw conv + BN + SiLU (+ squeeze) -> SE gate -> gate folded into the 1x1 projection's weights ->
    projection + BN (+ residual).  x: CL [B,1,H,W,C]."""
    L = _lib.lib()
    dev = plan.device
    B, _, H, W = x.dims
    Cm = x.C
    assert Cm % 8 == 0 and x.coff == 0
    OH, OW = math.ceil(H / stride), math.ceil(W / stride)
    pt, pl = same_pad(H, k, stride) // 2, same_pad(W, k, stride) // 2
    w, b = fold_bn(conv_dw.weight, None, bn_dw)
    wdw = w.reshape(Cm, k * k).t().contiguous()                # [K*K][C] fp32
    y = plan.alloc(B, 1, OH, OW, Cm)
    pool = torch.zeros(B, Cm, dtype=torch.int64, device=dev)      # squeeze sums, fixed point 2^-24 (deterministic)
    dw_fwd = _dw_entry(L)
    plan.add(FnOp(lambda st: dw_fwd(x.ptr, wdw.data_ptr(), b.data_ptr(), y.ptr, pool.data_ptr(), plan.lib_dtype, B,
                                    H, W, OH, OW, Cm, x.cstride, y.cstride, k, stride, pt, pl,
                                    _lib.ACT_SILU, st), name + ".dw", keep=(x, wdw, b, y, pool)))
    R = se.conv_reduce.out_channels
    w1 = se.conv_reduce.weight.detach().float().reshape(R, Cm).contiguous()
    b1 = se.conv_reduce.bias.detach().float().contiguous()
    w2t = se.conv_expand.weight.detach().float().reshape(Cm, R).t().contiguous()
    b2 = se.conv_expand.bias.detach().float().contiguous()
    wp, bp = fold_bn(conv_proj.weight, None, bn_proj)
    Cout = wp.shape[0]
    Cout_pad, Kp = _round_up(Cout, 16), plan.kpad_for(Cm)
    master = torch.zeros(Cout_pad, Kp, dtype=torch.float32, device=dev)
    master[:Cout, :Cm] = wp.reshape(Cout, Cm)
    if out is None:
        out = plan.alloc(B, 1, OH, OW, Cout)
    hidden = torch.empty(B, R, dtype=torch.float32, device=dev)
    # the gate is per image -> one projection-weight set per image, all images in ONE SE launch pair + ONE GEMM
    wbuf = torch.zeros(B, Cout_pad, Kp, dtype=plan.dtype, device=dev)
    se_fwd = L.occd_se_gate_fold_fwd
    plan.add(FnOp(lambda st: se_fwd(
        pool.data_ptr(), 1.0 / (OH * OW), w1.data_ptr(), b1.data_ptr(), w2t.data_ptr(), b2.data_ptr(),
        hidden.data_ptr(), master.data_ptr(), wbuf.data_ptr(), plan.lib_dtype, B, Cm, R, Cout_pad, Kp, st),
        name + ".se", keep=(pool, w1, b1, w2t, b2, hidden, master, wbuf)))
    plan.add(ConvOp([y], [(0, 0, 0, 0)], None, bp, (1, OH, OW), out0=out, res1=residual, weight_buf=wbuf,
                    weight_per_image=True, name=name + ".proj"))
    return out


class DepthwiseSeparableConv(nn.Module):
    def __init__(self, cin, cout, k, stride, se_chs):
        super().__init__()
        self.has_residual = stride == 1 and cin == cout
        self.k, self.stride = k, stride
        self.conv_dw = _conv(cin, cin, k, stride, groups=cin)
        self.bn1 = nn.BatchNorm2d(cin, eps=BN_EPS)
        self.act1 = nn.SiLU()
        self.se = SqueezeExcite(cin, se_chs)
        self.conv_pw = nn.Conv2d(cin, cout, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout, eps=BN_EPS)
        self.act2 = nn.Identity()

    def emit(self, plan, x, name="ds"):
        return _emit_dw_se_project(plan, x, self.conv_dw, self.bn1, self.se, self.conv_pw, self.bn2, self.k,
                                   self.stride, x if self.has_residual else None, name=name)


class InvertedResidual(nn.Module):
    def __init__(self, cin, cout, k, stride, expand, se_chs):
        super().__init__()
        mid = cin * expand
        self.has_residual = stride == 1 and cin == cout
        self.k, self.stride = k, stride
        self.conv_pw = nn.Conv2d(cin, mid, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(mid, eps=BN_EPS)
        self.act1 = nn.SiLU()
        self.conv_dw = _conv(mid, mid, k, stride, groups=mid)
        self.bn2 = nn.BatchNorm2d(mid, eps=BN_EPS)
        self.act2 = nn.SiLU()
        self.se = SqueezeExcite(mid, se_chs)
        self.conv_pwl = nn.Conv2d(mid, cout, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(cout, eps=BN_EPS)

    def emit(self, plan, x, name="ir"):
        w, b = fold_bn(self.conv_pw.weight, None, self.bn1)
        h = plan.conv(x, w.unsqueeze(2), b, act="silu", name=name + ".expand")
        return _emit_dw_se_project(plan, h, self.conv_dw, self.bn2, self.se, self.conv_pwl, self.bn3, self.k,
                                   self.stride, x if self.has_residual else None, name=name)


class GenEfficientNet(nn.Module):
    """geffnet GenEfficientNet layout; `emit_features` reproduces what Encoder.forward collects."""

    def __init__(self, name="tf_efficientnet_b7_ns", num_classes=1000):
        super().__init__()
        self.model_name = name
        stem, specs, head = block_specs(name)
        self.conv_stem = _conv(3, stem, 3, 2)
        self.bn1 = nn.BatchNorm2d(stem, eps=BN_EPS)
        self.act1 = nn.SiLU()
        stages = [[] for _ in ARCH]
        for (si, typ, cin, cout, k, stride, e, se) in specs:
            stages[si].append(DepthwiseSeparableConv(cin, cout, k, stride, se) if typ == "ds"
                              else InvertedResidual(cin, cout, k, stride, e, se))
        self.blocks = nn.Sequential(*[nn.Sequential(*s) for s in stages])
        self.conv_head = nn.Conv2d(specs[-1][3], head, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(head, eps=BN_EPS)
        self.act2 = nn.SiLU()
        self.global_pool = nn.AdaptiveAvgPool2d(1)
        self.classifier = nn.Linear(head, num_classes)

    def emit_features(self, plan, x):
        """x: CL image [B,1,H,W,3] -> dict {4,5,6,8,11: CL} = the entries of the reference's `features` list
        that DecoderBN consumes (unet2d.py:138-144): blocks[0],[1],[2],[4] outputs and conv_head's raw output
        (before bn2/act2, which the reference computes and discards)."""
        B, _, H, W = x.dims
        w, b = fold_bn(self.conv_stem.weight, None, self.bn1)
        k, s = 3, 2
        OH, OW = math.ceil(H / s), math.ceil(W / s)
        pt, pl = same_pad(H, k, s) // 2, same_pad(W, k, s) // 2
        from ..engine import conv_taps
        taps, ws = conv_taps(w.unsqueeze(2), (1, 1, 1), (0, pt, pl))
        y = plan.alloc(B, 1, OH, OW, w.shape[0])
        plan.add(ConvOp([x], taps, ws, b, (1, OH, OW), out0=y, act="silu", stride=(1, s, s), name="stem"))
        feats = {}
        for si, stage in enumerate(self.blocks):
            for bi, blk in enumerate(stage):
                y = blk.emit(plan, y, name="b%d.%d" % (si, bi))
            feats[4 + si] = y
        w = self.conv_head.weight.detach().float()
        feats[11] = plan.conv(y, w.unsqueeze(2), torch.zeros(w.shape[0], device=plan.device), name="conv_head")
        return feats
