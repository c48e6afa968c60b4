"""Drop-in for the reference `occdepth/models/unet3d_nyu.py` (UNet3D :16-110)."""
import numpy as np
import torch
import torch.nn as nn

from ._base import B200Module
from .CRP3D import CPMegaVoxels
from .modules import ASPP, Downsample, Process, SegmentationHead, SegmentationHeadCascadeCLS, Upsample  # noqa: F401


class UNet3D(B200Module):
    def __init__(self, class_num, norm_layer, feature, full_scene_size, n_relations=4, project_res=[],
                 context_prior=True, bn_momentum=0.1, cascade_cls=False, infer_mode=False):
        super(UNet3D, self).__init__()
        self.business_layer = []
        self.project_res = project_res
        self.cascade_cls = cascade_cls
        f4, f8, f16 = feature, feature * 2, feature * 4
        self.feature_1_4, self.feature_1_8, self.feature_1_16 = f4, f8, f16
        self.feature_1_4_dec, self.feature_1_8_dec, self.feature_1_16_dec = f4, f8, f16
        self.infer_mode = infer_mode

        def level(width):
            return nn.Sequential(Process(width, norm_layer, bn_momentum, dilations=[1, 2, 3]),
                                 Downsample(width, norm_layer, bn_momentum))

        self.process_1_4 = level(f4)
        self.process_1_8 = level(f8)
        self.up_1_16_1_8 = Upsample(f16, f8, norm_layer, bn_momentum)
        self.up_1_8_1_4 = Upsample(f8, f4, norm_layer, bn_momentum)
        head = SegmentationHeadCascadeCLS if self.cascade_cls else SegmentationHead
        self.ssc_head_1_4 = head(f4, f4, class_num, [1, 2, 3])
        self.context_prior = context_prior
        if context_prior:
            size_1_16 = tuple(int(np.ceil(i / 4)) for i in full_scene_size)
            self.CP_mega_voxels = CPMegaVoxels(f16, size_1_16, n_relations=n_relations, bn_momentum=bn_momentum)

    def emit(self, plan, x3d_1_4, classes=False, lut=None, confidence=False):
        """-> the forward's output dict, or with `classes` only the uint16 class map [B, X, Y, Z] of the ssc head
        (`confidence`: uint16 [2, B, X, Y, Z], the map and its float16 confidence bits, modules._classifier)"""
        res = {}
        x3d_1_8 = self.process_1_4[1].emit(plan, self.process_1_4[0].emit(plan, x3d_1_4))
        x3d_1_16 = self.process_1_8[1].emit(plan, self.process_1_8[0].emit(plan, x3d_1_8))
        if self.context_prior:
            ret = self.CP_mega_voxels.emit(plan, x3d_1_16)
            x3d_1_16 = ret["x"]
            for k in ret.keys():
                res[k] = ret[k]
        x3d_up_1_8 = self.up_1_16_1_8.emit(plan, x3d_1_16, skip=x3d_1_8)
        x3d_up_1_4 = self.up_1_8_1_4.emit(plan, x3d_up_1_8, skip=x3d_1_4)
        if classes:
            out = self.ssc_head_1_4.emit(plan, x3d_up_1_4, classes=True, lut=lut, confidence=confidence)
            return out[0] if self.cascade_cls else out
        if not self.infer_mode:
            res["x3d_l1"] = x3d_up_1_4
            res["x3d_l2"] = x3d_up_1_8
            res["x3d_l3"] = x3d_1_16
        if self.cascade_cls:
            ssc_logit_full, ssc_logit_full_occ = self.ssc_head_1_4.emit(plan, x3d_up_1_4)
            res["ssc_logit"] = ssc_logit_full
            if not self.infer_mode:
                res["occ_logit"] = ssc_logit_full_occ
        else:
            res["ssc_logit"] = self.ssc_head_1_4.emit(plan, x3d_up_1_4)
        return res

    def forward(self, input_dict):
        return self._run_planar(input_dict["x3d"])
