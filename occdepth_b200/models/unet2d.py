"""Drop-in for the reference `occdepth/models/unet2d.py`: UpSampleBN :24-46, DecoderBN :49-180, Encoder :183-196,
UNet2D :199-255.

The decoder's `torch.cat([up_x, skip])` is never materialised.  Bilinear resizing commutes with a channel mix, so on
the wide levels (split_pays) UpSampleBN's first 3x3 conv is split by input half: the up half runs as ONE 1x1 GEMM on
the coarse map producing all nine taps' products (tap-major, pack_tap_weights), occd_upsample_tapsum_ac resizes them
and sums them on the fine grid (the fine grid's zero padding becomes an in-bounds mask), and the skip half is an
ordinary 3x3 conv whose pre-activation the tap sum adds to before the LeakyReLU.  That executes about a quarter of the
up half's reference MACs (DESIGN.md section 4.5).  On the narrow levels the resized map is materialised and the 3x3
conv reads it and the skip as two TMA sources into one accumulator.
"""
import os

import torch
import torch.nn as nn

from .. import _lib
from ..engine import ACT, CL, ConvOp, FnOp, conv_taps, fold_bn
from ._base import B200Module
from .efficientnet import GenEfficientNet

MODEL_NAME = "tf_efficientnet_b3_ns"
MODEL_CHANNELS = {
    "tf_efficientnet_b3_ns": [3, 24, 32, 48, 136],
    "tf_efficientnet_b4_ns": [3, 24, 32, 56, 160],
    "tf_efficientnet_b5_ns": [3, 32, 40, 64, 176],
    "tf_efficientnet_b7_ns": [3, 32, 48, 80, 224],
}
NUM_FEATURES = {
    "tf_efficientnet_b3_ns": 1536,
    "tf_efficientnet_b4_ns": 1792,
    "tf_efficientnet_b5_ns": 2048,
    "tf_efficientnet_b7_ns": 2560,
}


def pack_tap_weights(w_up):
    """conv1's up-half weights [Cout, C_up, 3, 3] -> the coarse GEMM's [9 * Cp, C_up] matrix in tap-major blocks: row
    t * Cp + o holds w_up[o, :, dy + 1, dx + 1], t = (dy + 1) * 3 + (dx + 1); Cp = Cout rounded up to 8 (so every
    tap's channel block starts on a vector), padding rows zero."""
    co, ci = w_up.shape[:2]
    cp = (co + 7) // 8 * 8
    wt = w_up.new_zeros(9, cp, ci)
    wt[:, :co] = w_up.permute(2, 3, 0, 1).reshape(9, co, ci)
    return wt.reshape(9 * cp, ci)


SPLIT_MIN_COUT = 192


def split_pays(co):
    """Whether UpSampleBN's conv1 runs split (coarse tap GEMM + tap sum + skip conv).  The split saves 3/4 of the up
    half's MACs but writes and reads the nine per-tap products (about 1.1x the resized map) and a pre-activation map.
    Every decoder level has C_up = 2 * Cout, so MACs saved per fine pixel grow as Cout^2 and the added bytes as Cout.
    Measured on the B7 decoder (H100, tf32, DESIGN.md section 7): 1.8x faster at Cout 1280, 1.6x at 640, 1.4x at 320,
    even at 160, 0.7x at 80."""
    return co >= SPLIT_MIN_COUT


class UpSampleBN(B200Module):
    def __init__(self, skip_input, output_features):
        super(UpSampleBN, self).__init__()
        self._net = nn.Sequential(
            nn.Conv2d(skip_input, output_features, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(output_features),
            nn.LeakyReLU(),
            nn.Conv2d(output_features, output_features, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(output_features),
            nn.LeakyReLU())

    def emit(self, plan, x, concat_with, name="up"):
        """conv1(cat(U(x), skip)) as  act(conv1_skip(skip) + bias + tapsum(Y)),  Y = W_up x on the coarse grid, where
        that pays (split_pays); else the resize is materialised and conv1 reads it and the skip as two sources."""
        B, _, h, w = x.dims
        _, _, OH, OW = concat_with.dims
        w1, b1 = fold_bn(self._net[0].weight, self._net[0].bias, self._net[1])
        assert w1.shape[1] == x.C + concat_with.C
        co = w1.shape[0]
        if split_pays(co):
            y = self._emit_conv1_split(plan, x, concat_with, w1, b1, name)
        else:
            up = plan.alloc(B, 1, OH, OW, x.C)
            up_fwd = _lib.lib().occd_upsample_bilinear_ac
            plan.add(FnOp(lambda st: up_fwd(x.ptr, up.ptr, plan.lib_dtype, B, h, w, OH, OW, x.C, x.cstride, x.coff,
                                            up.cstride, up.coff, st),
                          name + ".bilinear", keep=(x, up)))
            t0, ws0 = conv_taps(w1[:, : x.C].unsqueeze(2), (1, 1, 1), (0, 1, 1), src=0)
            t1, ws1 = conv_taps(w1[:, x.C:].unsqueeze(2), (1, 1, 1), (0, 1, 1), src=1)
            y = plan.alloc(B, 1, OH, OW, co)
            plan.add(ConvOp([up, concat_with], t0 + t1, ws0 + ws1, b1, (1, OH, OW), out0=y, act="leaky",
                            name=name + ".conv1"))
        w2, b2 = fold_bn(self._net[3].weight, self._net[3].bias, self._net[4])
        return plan.conv(y, w2.unsqueeze(2), b2, padding=(0, 1, 1), act="leaky", name=name + ".conv2")

    @staticmethod
    def _emit_conv1_split(plan, x, concat_with, w1, b1, name):
        B, _, h, w = x.dims
        _, _, OH, OW = concat_with.dims
        co = w1.shape[0]
        wy = pack_tap_weights(w1[:, : x.C])
        tap_stride = wy.shape[0] // 9
        # the up half: nine per-tap 1x1 products in one GEMM on the coarse map, kept unrounded (they only feed a sum)
        ys = plan.alloc(B, 1, h, w, wy.shape[0])
        taps = plan.add(ConvOp([x], [(0, 0, 0, 0)], [wy], torch.zeros(wy.shape[0], device=wy.device), (1, h, w),
                               out0=ys, out0_exact=True, name=name + ".taps"))
        # the skip half: pre-activation (bias included), exact; the tap sum adds to it, activates and rounds in place
        t1, ws1 = conv_taps(w1[:, x.C:].unsqueeze(2), (1, 1, 1), (0, 1, 1), src=0)
        y = plan.alloc(B, 1, OH, OW, co)
        plan.add(ConvOp([concat_with], t1, ws1, b1, (1, OH, OW), out0=y, out0_exact=True, name=name + ".conv1"))
        tapsum = _lib.lib().occd_upsample_tapsum_ac
        # FLOP bookkeeping: the tap sum carries the reference up half's 2*MACs that the coarse GEMM did not execute
        up_flops = 2 * B * OH * OW * co * 9 * x.C
        plan.add(FnOp(lambda st: tapsum(ys.ptr, y.ptr, y.ptr, plan.lib_dtype, B, h, w, OH, OW, co, ys.cstride, ys.coff,
                                        tap_stride, y.cstride, y.coff, y.cstride, y.coff, ACT["leaky"], st),
                      name + ".tapsum", keep=(ys, y), flops=max(up_flops - taps.flops, 0)))
        return y

    def forward(self, x, concat_with):
        raise RuntimeError("UpSampleBN: use UNet2D.forward (the block has two inputs and is planned as a whole)")


class DecoderBN(B200Module):
    def __init__(self, num_features, bottleneck_features, out_feature, use_decoder=True, backbone_2d_name=None,
                 return_up_feats=None):
        super(DecoderBN, self).__init__()
        features = int(num_features)
        self.use_decoder = use_decoder
        self.backbone_2d_name = backbone_2d_name
        self.return_up_feats = return_up_feats
        # 1x1 conv WITH padding=1: a (h+2)x(w+2) map whose border is bias only (reference unet2d.py:65-67)
        self.conv2 = nn.Conv2d(bottleneck_features, features, kernel_size=1, stride=1, padding=1)
        scales = (1, 2, 4, 8, 16)
        for s in scales:                                   # decoder widths features/32 .. features/2
            setattr(self, "out_feature_1_%d" % s, out_feature)
        for s, div in zip(scales[::-1], (2, 4, 8, 16, 32)):
            setattr(self, "feature_1_%d" % s, features // div)
        if not self.use_decoder:
            self.resize_output_1_1 = nn.Conv2d(3, out_feature, kernel_size=1)
            self.resize_output_1_2 = nn.Conv2d(32, out_feature * 2, kernel_size=1)
            self.resize_output_1_4 = nn.Conv2d(48, out_feature * 4, kernel_size=1)
            return
        # registration order == the reference's (state_dict order): the five 1x1 heads, then up16 .. up1
        for s in scales:
            if self.return_up_feats <= s:
                setattr(self, "resize_output_1_%d" % s,
                        nn.Conv2d(getattr(self, "feature_1_%d" % s), out_feature, kernel_size=1))
        skip_ch = MODEL_CHANNELS[self.backbone_2d_name]     # [image, blocks[0], blocks[1], blocks[2], blocks[4]]
        below = features                                    # channels coming up from the coarser level
        for s, skip in zip(scales[::-1], skip_ch[::-1]):
            width = getattr(self, "feature_1_%d" % s)
            if self.return_up_feats <= s:
                setattr(self, "up%d" % s, UpSampleBN(skip_input=below + skip, output_features=width))
            below = width

    def emit(self, plan, features, outs=None):
        """features: {0: image CL, 4,5,6,8,11: encoder CLs}; outs: optional {"1_s": CL} destinations.
        Returns {"1_16","1_8","1_4","1_2","1_1"} channels-last (reference DecoderBN.forward :137-165)."""
        if not self.use_decoder:
            raise NotImplementedError("DecoderBN(use_decoder=False) is not on the reference's configured path")
        outs = outs or {}

        def resize(conv, x, key):
            w = conv.weight.detach().float()
            return plan.conv(x, w.unsqueeze(2), conv.bias.detach().float(), out=outs.get(key), name="resize_" + key)

        c2 = self.conv2
        x_d0 = plan.conv(features[11], c2.weight.detach().float().unsqueeze(2), c2.bias.detach().float(),
                         padding=(0, 1, 1), name="dec.conv2")   # 1x1 conv with padding=1 (unet2d.py:65-67)
        res = {}
        x = self.up16.emit(plan, x_d0, features[8], "up16")
        res["1_16"] = resize(self.resize_output_1_16, x, "1_16")
        if self.return_up_feats <= 8:
            x = self.up8.emit(plan, x, features[6], "up8")
            res["1_8"] = resize(self.resize_output_1_8, x, "1_8")
        if self.return_up_feats <= 4:
            x = self.up4.emit(plan, x, features[5], "up4")
            res["1_4"] = resize(self.resize_output_1_4, x, "1_4")
        if self.return_up_feats <= 2:
            x = self.up2.emit(plan, x, features[4], "up2")
            res["1_2"] = resize(self.resize_output_1_2, x, "1_2")
        if self.return_up_feats <= 1:
            x = self.up1.emit(plan, x, features[0], "up1")
            res["1_1"] = resize(self.resize_output_1_1, x, "1_1")
        return res

    def forward(self, features):
        raise RuntimeError("DecoderBN: use UNet2D.forward (planned as a whole)")


class Encoder(B200Module):
    def __init__(self, backend):
        super(Encoder, self).__init__()
        self.original_model = backend

    def emit(self, plan, x):
        feats = self.original_model.emit_features(plan, x)
        feats[0] = x
        return feats

    def forward(self, x):
        raise RuntimeError("Encoder: use UNet2D.forward (planned as a whole)")


class UNet2D(B200Module):
    def __init__(self, backend, num_features, out_feature, use_decoder=True, backbone_2d_name=None,
                 return_up_feats=1):
        super(UNet2D, self).__init__()
        self.use_decoder = use_decoder
        self.encoder = Encoder(backend)
        self.decoder = DecoderBN(out_feature=out_feature, use_decoder=use_decoder, bottleneck_features=num_features,
                                 num_features=num_features, backbone_2d_name=backbone_2d_name,
                                 return_up_feats=return_up_feats)

    def emit(self, plan, x, outs=None):
        return self.decoder.emit(plan, self.encoder.emit(plan, x), outs)

    def forward(self, x, **kwargs):
        return self._run_planar(x, squeeze_d=True)

    def get_encoder_params(self):  # lr/10 learning rate
        return self.encoder.parameters()

    def get_decoder_params(self):  # lr learning rate
        return self.decoder.parameters()

    @classmethod
    def build(cls, **kwargs):
        basemodel_name = kwargs["backbone_2d_name"]
        num_features = NUM_FEATURES[basemodel_name]
        print("Loading base model {}...".format(basemodel_name), end="")
        # the reference downloads pretrained geffnet weights here (torch.hub); offline we build the same
        # architecture with default init -- load a checkpoint's state_dict to get trained weights
        basemodel = GenEfficientNet(basemodel_name)
        print("Done.")
        print("Removing last two layers (global_pool & classifier).")
        basemodel.global_pool = nn.Identity()
        basemodel.classifier = nn.Identity()
        print("Building Encoder-Decoder model..", end="")
        m = cls(basemodel, num_features=num_features, **kwargs)
        print("Done.")
        print("INFO: return_up_feats set to : {}.".format(kwargs["return_up_feats"]))
        return m
