"""Drop-in for the reference `occdepth/models/unet3d_kitti.py` (UNet3D :14-126)."""
import torch
import torch.nn as nn

from ._base import B200Module
from .CRP3D import CPMegaVoxels
from .modules import (Convblock3d, Downsample, Process, SegmentationHead, SegmentationHeadCascadeCLS,
                      SegmentationHeadOccludedCLS, Upsample)


class UNet3D(B200Module):
    def __init__(self, class_num, norm_layer, full_scene_size, feature, project_scale, context_prior=None,
                 bn_momentum=0.1, cascade_cls=False, occluded_cls=False, infer_mode=False):
        super(UNet3D, self).__init__()
        self.business_layer = []
        self.project_scale = project_scale
        self.full_scene_size = full_scene_size
        self.feature = feature
        self.cascade_cls = cascade_cls
        self.occluded_cls = occluded_cls
        self.infer_mode = infer_mode
        f = self.feature
        size_l3 = tuple(int(s / project_scale) // 4 for s in self.full_scene_size)      # the 1/4 grid of the lift grid
        heads = {True: SegmentationHeadCascadeCLS, False: SegmentationHead}
        dil = [1, 2, 3]

        def level(width):
            return nn.Sequential(Process(width, norm_layer, bn_momentum, dilations=[1, 2, 3]),
                                 Downsample(width, norm_layer, bn_momentum))

        # encoder: two (Process, Downsample) levels; decoder: transposed convs back up, skip adds in forward
        self.process_l1 = level(f)
        self.process_l2 = level(f * 2)
        self.up_13_l2 = Upsample(f * 4, f * 2, norm_layer, bn_momentum)
        self.up_12_l1 = Upsample(f * 2, f, norm_layer, bn_momentum)
        # lift grid == full grid (project_scale 1): stride-1 block; otherwise one more x2 up-sampling to full res
        self.up_l1_lfull = (Convblock3d(f, f // 2, norm_layer, bn_momentum, stride=1) if self.project_scale == 1
                            else Upsample(f, f // 2, norm_layer, bn_momentum))
        self.ssc_head = heads[bool(self.cascade_cls)](f // 2, f // 2, class_num, dil)
        if self.occluded_cls:
            self.occluded_head = SegmentationHeadOccludedCLS(f // 2, f // 2, class_num, dil)
        self.context_prior = context_prior
        if context_prior:
            self.CP_mega_voxels = CPMegaVoxels(f * 4, size_l3, bn_momentum=bn_momentum)

    def emit(self, plan, x3d_l1, classes=False, lut=None, confidence=False, probabilities=False):
        """-> the forward's output dict, or with `classes` only the uint16 class map [B, X, Y, Z] of the ssc head
        (`confidence`: uint16 [2, B, X, Y, Z], the map and its float16 confidence bits; `probabilities`: the map
        and every class's float16 probability bits, uint16 [(1 + C) * B, X, Y, Z]; modules._classifier)
        (the occluded head, whose logits nothing then reads, is not planned)"""
        res = {}
        x3d_l2 = self.process_l1[1].emit(plan, self.process_l1[0].emit(plan, x3d_l1))
        x3d_l3 = self.process_l2[1].emit(plan, self.process_l2[0].emit(plan, x3d_l2))
        if self.context_prior:
            ret = self.CP_mega_voxels.emit(plan, x3d_l3)
            x3d_l3 = ret["x"]
            for k in ret.keys():
                res[k] = ret[k]
        x3d_up_l2 = self.up_13_l2.emit(plan, x3d_l3, skip=x3d_l2)
        x3d_up_l1 = self.up_12_l1.emit(plan, x3d_up_l2, skip=x3d_l1)
        x3d_up_lfull = self.up_l1_lfull.emit(plan, x3d_up_l1)
        if classes:
            out = self.ssc_head.emit(plan, x3d_up_lfull, classes=True, lut=lut, confidence=confidence,
                                     probabilities=probabilities)
            return out[0] if self.cascade_cls else out
        if not self.infer_mode:
            res["x3d_l1"] = x3d_up_l1
            res["x3d_l2"] = x3d_up_l2
            res["x3d_l3"] = x3d_l3
        if self.cascade_cls:
            ssc_logit_full, ssc_logit_full_occ = self.ssc_head.emit(plan, x3d_up_lfull)
            res["ssc_logit"] = ssc_logit_full
            if not self.infer_mode:
                res["occ_logit"] = ssc_logit_full_occ
        else:
            res["ssc_logit"] = self.ssc_head.emit(plan, x3d_up_lfull)
        if self.occluded_cls:
            occluded_logit_full = self.occluded_head.emit(plan, x3d_up_lfull)
            if not self.infer_mode:
                res["occluded_logit"] = occluded_logit_full
        return res

    def forward(self, input_dict):
        return self._run_planar(input_dict["x3d"])
