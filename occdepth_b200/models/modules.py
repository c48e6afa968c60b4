"""Drop-in for the reference `occdepth/models/modules.py` (3D building blocks), forward on sm_90a kernels.

ASPP :6-48, SegmentationHead :51-106, SegmentationHeadCascadeCLS :109-175, SegmentationHeadOccludedCLS
:178-235, Process :258-275, Upsample :278-296, Convblock3d :299-317, Downsample :320-344.
"""
import torch
import torch.nn as nn

from .. import _lib
from ..engine import FnOp, fold_bn
from ._base import B200Module
from .DDR import Bottleneck3D


def _emit_aspp(plan, m, x, out=None, name="aspp"):
    """relu( sum_i bn2_i(conv2_i(relu(bn1_i(conv1_i(x))))) + x ): 3 launches for conv1, ONE launch for the three
    conv2 branches (81 taps, one accumulator) with the residual + ReLU in its epilogue."""
    ts, ws, b2s, bs = [], [], [], None
    for i, dl in enumerate(m.conv_list):
        w, b = fold_bn(m.conv1[i].weight, m.conv1[i].bias, m.bn1[i])
        ts.append(plan.conv(x, w, b, padding=dl, dilation=dl, act="relu", name="%s.conv1.%d" % (name, i)))
        w2, b2 = fold_bn(m.conv2[i].weight, m.conv2[i].bias, m.bn2[i])
        ws.append(w2)
        b2s.append(b2)
        bs = b2 if bs is None else bs + b2
    from ..engine import default_impl
    if x.C <= 64 and default_impl() is None:
        # few channels (the full-resolution head): three halo-tile launches chained through the residual input
        # (partial sums stored as bf16) beat one 81-tap launch of the per-tap kernel by ~2.5x
        y = None
        n = len(ts)
        for i, dl in enumerate(m.conv_list):
            last = i == n - 1
            # the partial sums only feed the next launch's epilogue add (never an MMA operand): unrounded in tf32 mode
            y = plan.conv(ts[i], ws[i], b2s[i], padding=dl, dilation=dl, act="relu" if last else "none", res1=y,
                          res2=x if last else None, out=out if last else None, name="%s.conv2.%d" % (name, i),
                          out0_exact=not last)
        return y
    return plan.conv_multi(ts, ws, bs, list(m.conv_list), list(m.conv_list), act="relu", res1=x, out=out,
                           name=name + ".conv2")


def _aspp_params(self, planes, dilations_conv_list):
    self.conv_list = dilations_conv_list
    self.conv1 = nn.ModuleList(
        [nn.Conv3d(planes, planes, kernel_size=3, padding=dil, dilation=dil, bias=False) for dil in dilations_conv_list])
    self.bn1 = nn.ModuleList([nn.BatchNorm3d(planes) for dil in dilations_conv_list])
    self.conv2 = nn.ModuleList(
        [nn.Conv3d(planes, planes, kernel_size=3, padding=dil, dilation=dil, bias=False) for dil in dilations_conv_list])
    self.bn2 = nn.ModuleList([nn.BatchNorm3d(planes) for dil in dilations_conv_list])
    self.relu = nn.ReLU()


def _planar_out(plan, x, C_):
    B, D, H, W = x.dims
    return torch.empty(B, C_, D, H, W, dtype=torch.float32, device=plan.device)


def _classifier(plan, x, w, b, name, classes, lut, res1=None, confidence=False):
    """the head's last conv: fp32 planar logits [B, n_classes, D, H, W], or (classes) their uint16 arg-max map
    [B, D, H, W] (label ids lut[class] when lut is given) written by the same epilogue instead; with `confidence`
    uint16 [2, B, D, H, W]: that map, then the float16 bits of each voxel's top-class softmax probability"""
    if classes:
        B, D, H, W = x.dims
        shape, mode = ((2, B, D, H, W), "classes_conf") if confidence else ((B, D, H, W), "classes")
        out = torch.empty(shape, dtype=torch.uint16, device=plan.device)
        plan.conv(x, w, b, padding=1, res1=res1, out1=out, out1_mode=mode, lut=lut, no_out0=True, name=name)
        return out
    out = _planar_out(plan, x, w.shape[0])
    plan.conv(x, w, b, padding=1, res1=res1, out1=out, out1_mode="planar", no_out0=True, name=name)
    return out


class ASPP(B200Module):
    def __init__(self, planes, dilations_conv_list):
        super().__init__()
        _aspp_params(self, planes, dilations_conv_list)

    def emit(self, plan, x, out=None):
        return _emit_aspp(plan, self, x, out)

    def forward(self, x_in):
        return self._run_planar(x_in)


class SegmentationHead(B200Module):
    def __init__(self, inplanes, planes, nbr_classes, dilations_conv_list):
        super().__init__()
        self.conv0 = nn.Conv3d(inplanes, planes, kernel_size=3, padding=1, stride=1)
        _aspp_params(self, planes, dilations_conv_list)
        self.conv_classes = nn.Conv3d(planes, nbr_classes, kernel_size=3, padding=1, stride=1)

    def emit(self, plan, x, classes=False, lut=None, confidence=False):
        """-> fp32 planar logits [B, n_classes, X, Y, Z] (written directly by the last conv's epilogue), or with
        `classes` their uint16 class map [B, X, Y, Z] (`confidence`: see _classifier)"""
        w, b = fold_bn(self.conv0.weight, self.conv0.bias, None)
        x0 = plan.conv(x, w, b, padding=1, act="relu", name="head.conv0")
        x1 = _emit_aspp(plan, self, x0, name="head.aspp")
        w, b = fold_bn(self.conv_classes.weight, self.conv_classes.bias, None)
        return _classifier(plan, x1, w, b, "head.conv_classes", classes, lut, confidence=confidence)

    def forward(self, x_in):
        return self._run_planar(x_in)


class SegmentationHeadCascadeCLS(B200Module):
    def __init__(self, inplanes, planes, nbr_classes, dilations_conv_list):
        super().__init__()
        self.conv0 = nn.Conv3d(inplanes, planes, kernel_size=3, padding=1, stride=1)
        _aspp_params(self, planes, dilations_conv_list)
        occ_classes = 2
        self.conv_classes = nn.Conv3d(planes + occ_classes, nbr_classes, kernel_size=3, padding=1, stride=1)
        self.occ_classes = nn.Conv3d(planes, occ_classes, kernel_size=3, padding=1, stride=1)
        self.softmax = nn.Softmax(dim=1)

    def emit(self, plan, x, classes=False, lut=None, confidence=False):
        """-> (ssc logits, occupancy logits), fp32 planar; with `classes` the ssc output is the uint16 class map
        [B, X, Y, Z] (the occupancy logits still feed the softmax; `confidence`: see _classifier)"""
        planes = self.conv0.out_channels
        w, b = fold_bn(self.conv0.weight, self.conv0.bias, None)
        x0 = plan.conv(x, w, b, padding=1, act="relu", name="head.conv0")
        B, D, H, W = x0.dims
        x1 = _emit_aspp(plan, self, x0, name="head.aspp")
        w, b = fold_bn(self.occ_classes.weight, self.occ_classes.bias, None)
        x_occ = _planar_out(plan, x1, 2)
        plan.conv(x1, w, b, padding=1, out1=x_occ, out1_mode="planar", no_out0=True, name="head.occ_classes")
        # torch.cat([x_in, softmax(x_occ)]) is never built: conv_classes is split along its input channels into
        # the `planes`-channel part (k-chunk of 32/64 channels) and the 2 softmax channels (k-chunk of 16); the
        # second launch adds the first one's result in its epilogue and writes the NCDHW fp32 logits
        L = _lib.lib()
        S = D * H * W
        sm = plan.alloc(B, D, H, W, 2)
        plan.add(FnOp(lambda st: L.occd_softmax_planar_to_cl(x_occ.data_ptr(), sm.ptr, plan.lib_dtype, B, 2, S,
                                                            sm.cstride, sm.coff, st), "occd_softmax_planar_to_cl",
                      keep=(x_occ, sm)))
        w, b = fold_bn(self.conv_classes.weight, self.conv_classes.bias, None)
        # `part` only feeds the second launch's epilogue add (never an MMA operand): stored unrounded in tf32 mode
        part = plan.conv(x1, w[:, :planes].contiguous(), b, padding=1, name="head.conv_classes.a", out0_exact=True)
        logits = _classifier(plan, sm, w[:, planes:].contiguous(), torch.zeros_like(b), "head.conv_classes.b", classes,
                             lut, res1=part, confidence=confidence)
        return logits, x_occ

    def forward(self, x_in):
        return self._run_planar(x_in)


class SegmentationHeadOccludedCLS(B200Module):
    def __init__(self, inplanes, planes, nbr_classes, dilations_conv_list):
        super().__init__()
        self.conv0 = nn.Conv3d(inplanes, planes, kernel_size=3, padding=1, stride=1)
        _aspp_params(self, planes, dilations_conv_list)
        occ_classes = 2
        self.occ_classes = nn.Conv3d(planes, occ_classes, kernel_size=3, padding=1, stride=1)

    def emit(self, plan, x):
        w, b = fold_bn(self.conv0.weight, self.conv0.bias, None)
        x0 = plan.conv(x, w, b, padding=1, act="relu", name="occl.conv0")
        x1 = _emit_aspp(plan, self, x0, name="occl.aspp")
        w, b = fold_bn(self.occ_classes.weight, self.occ_classes.bias, None)
        x_occ = _planar_out(plan, x1, 2)
        plan.conv(x1, w, b, padding=1, out1=x_occ, out1_mode="planar", no_out0=True, name="occl.occ_classes")
        return x_occ

    def forward(self, x_in):
        return self._run_planar(x_in)


class Process(B200Module):
    def __init__(self, feature, norm_layer, bn_momentum, dilations=[1, 2, 3]):
        super(Process, self).__init__()
        self.main = nn.Sequential(
            *[Bottleneck3D(feature, feature // 4, bn_momentum=bn_momentum, norm_layer=norm_layer,
                           dilation=[i, i, i]) for i in dilations])

    def emit(self, plan, x, out=None):
        n = len(self.main)
        for i, blk in enumerate(self.main):
            x = blk.emit(plan, x, out=out if i == n - 1 else None)
        return x

    def forward(self, x):
        return self._run_planar(x)


def _fold_bn_transposed(conv, bn):
    """ConvTranspose3d weight is [Cin, Cout, k, k, k]: BatchNorm scale applies along dim 1."""
    w = conv.weight.detach().float()
    co = w.shape[1]
    b = conv.bias.detach().float() if conv.bias is not None else torch.zeros(co, device=w.device)
    scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    return w * scale.view(1, co, 1, 1, 1), (b - bn.running_mean.detach().float()) * scale + bn.bias.detach().float()


class Upsample(B200Module):
    def __init__(self, in_channels, out_channels, norm_layer, bn_momentum):
        super(Upsample, self).__init__()
        self.main = nn.Sequential(
            nn.ConvTranspose3d(in_channels, out_channels, kernel_size=3, stride=2, padding=1, dilation=1,
                               output_padding=1),
            norm_layer(out_channels, momentum=bn_momentum),
            nn.ReLU())

    def emit(self, plan, x, skip=None):
        """relu(bn(convT(x))) [+ skip]: the skip add of unet3d_*.py rides in the epilogue (post-activation)."""
        w, b = _fold_bn_transposed(self.main[0], self.main[1])
        return plan.conv_transpose_k3s2(x, w, b, act="relu", res_post=skip, name="up")

    def forward(self, x):
        return self._run_planar(x)


class Convblock3d(B200Module):
    def __init__(self, in_channels, out_channels, norm_layer, bn_momentum, stride=1):
        super(Convblock3d, self).__init__()
        self.main = nn.Sequential(
            nn.ConvTranspose3d(in_channels, out_channels, kernel_size=3, stride=stride, padding=1, dilation=1,
                               output_padding=0),
            norm_layer(out_channels, momentum=bn_momentum),
            nn.ReLU())
        self.stride = stride

    def emit(self, plan, x):
        if self.stride != 1:
            raise NotImplementedError("Convblock3d: only stride 1 is on the reference's path (unet3d_kitti.py:63-66)")
        w, b = _fold_bn_transposed(self.main[0], self.main[1])
        # stride-1 transposed conv == conv with the flipped kernel and swapped channel axes
        wc = w.flip(2, 3, 4).permute(1, 0, 2, 3, 4).contiguous()
        return plan.conv(x, wc, b, padding=1, act="relu", name="convblock")

    def forward(self, x):
        return self._run_planar(x)


class Downsample(B200Module):
    def __init__(self, feature, norm_layer, bn_momentum, expansion=8):
        super(Downsample, self).__init__()
        self.main = Bottleneck3D(
            feature, feature // 4, bn_momentum=bn_momentum, expansion=expansion, stride=2,
            downsample=nn.Sequential(
                nn.AvgPool3d(kernel_size=2, stride=2),
                nn.Conv3d(feature, int(feature * expansion / 4), kernel_size=1, stride=1, bias=False),
                norm_layer(int(feature * expansion / 4), momentum=bn_momentum)),
            norm_layer=norm_layer)

    def emit(self, plan, x, out=None):
        return self.main.emit(plan, x, out=out)

    def forward(self, x):
        return self._run_planar(x)
