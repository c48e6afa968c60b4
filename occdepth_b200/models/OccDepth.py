"""Drop-in for the reference `occdepth/models/OccDepth.py` (class OccDepth, forward path :31-376).

Same constructor, same `forward(batch) -> dict`, same state_dict keys.  The forward is one planned sequence of
sm_90a launches: both stereo views go through the 2D UNet as one batch, the 4-scale / 2-view Stereo-SFA lift
is a single fused kernel writing the channels-last voxel grid the 3D UNet consumes, and the logits are written
in the reference's NCDHW fp32 layout by the last convolution's epilogue.
Evaluation (`test_step` / `validation_step` and their epoch-end hooks) counts the SSC metrics of `predict_classes` on
the device (occdepth_b200.metrics); with OCCDEPTH_EVAL_LOSSES=1 the steps also log the reference's losses, formed on
the device (occdepth_b200.losses).  Training (`training_step`, backward, optimisers; OccDepth.py:535-538) is out of
scope.
"""
import os
from collections.abc import Mapping

import torch
import torch.nn as nn

from .. import _lib
from ..engine import CL, FnOp, Plan, _round_up, require_cuda
from ..losses import step_losses
from ..metrics import SSCMetrics
from ._base import B200Module, _to_planar
from .SFA import SFA, lift_multiscale
from .unet2d import UNet2D
from .unet3d_kitti import UNet3D as UNet3DKitti
from .unet3d_nyu import UNet3D as UNet3DNYU
from .modules import split_probs

try:  # the reference derives from pl.LightningModule; use it when present so Trainer-based scripts keep working
    import pytorch_lightning as pl
    _Base = pl.LightningModule
except Exception:  # noqa: BLE001
    class _Base(nn.Module):
        def save_hyperparameters(self, *a, **k):
            pass

        def log(self, *a, **k):
            pass


def feature_hw(img_h, img_w, scale):
    """spatial size of the "1_scale" feature map (TF-SAME stride-2 stages: ceil division per halving)"""
    h, w, s = img_h, img_w, 1
    while s < scale:
        h, w, s = (h + 1) // 2, (w + 1) // 2, s * 2
    return h, w


def _check_class_request(who, classes, confidence, probabilities):
    """the refusals of probabilities=True (every class's softmax probability beside the class map)"""
    if not probabilities:
        return
    if not classes:
        raise ValueError("OccDepth.%s: probabilities=True are the class map's probabilities (classes=True)" % who)
    if confidence:
        raise ValueError("OccDepth.%s: probabilities=True already hold the confidence (the probability at the map's "
                         "class); ask for one of the two" % who)


def _get(config, name, default=None):
    try:
        return getattr(config, name)
    except (AttributeError, KeyError):
        return default


class OccDepth(_Base, B200Module):
    def __init__(self, class_names, class_weights, class_weights_occ=None, full_scene_size=None, project_res=[],
                 config=None, infer_mode=False):
        super().__init__()
        self.project_res = project_res
        self.full_scene_size = full_scene_size
        self.class_names = class_names
        self.class_weights = class_weights
        self.class_weights_occ = class_weights_occ
        self.dataset = config.dataset
        self.project_scale = config.project_scale
        self.n_relations = config.n_relations
        self.context_prior = config.context_prior
        self.n_classes = config.n_classes
        self.feature = config.feature
        self.feature_2d_oc = config.feature_2d_oc
        self.trans_2d_to_3d = config.trans_2d_to_3d
        self.cascade_cls = config.cascade_cls
        self.occluded_cls = config.occluded_cls
        self.multi_view_mode = _get(config, "multi_view_mode", True)
        self.share_2d_backbone_gradient = _get(config, "share_2d_backbone_gradient", False)
        print("INFO: Use cascade cls: {}".format(self.cascade_cls))
        print("INFO: Use occluded cls: {}".format(self.occluded_cls))
        self.infer_mode = infer_mode
        if self.infer_mode:
            self.context_prior = False
        # the loss switches of OccDepth.step (OccDepth.py:48-69, 96, 138-147); the losses run when
        # OCCDEPTH_EVAL_LOSSES=1.  The drop-in never trains, so cur_batch stays 0 and the sem-scal decay factor is 1
        self.relation_loss = _get(config, "relation_loss", False)
        self.CE_ssc_loss = _get(config, "CE_ssc_loss", False)
        self.sem_scal_loss = _get(config, "sem_scal_loss", False)
        self.geo_scal_loss = _get(config, "geo_scal_loss", False)
        self.fp_loss = _get(config, "fp_loss", False)
        self.frustum_size = _get(config, "frustum_size", 4)
        self.sem_step_decay_loss = _get(config, "sem_step_decay_loss", False)
        self.depth_loss_w = _get(config, "depth_loss_weight", 1.0)
        batch_size = _get(config, "batch_size_per_gpu", 1) * _get(config, "n_gpus", 1)
        self.total_batch = ((3834 if config.dataset == "kitti" else 795) // batch_size) * 30
        self.cur_batch = 0
        self.use_stereo_depth_gt = _get(config, "use_stereo_depth_gt", False)
        self.use_lidar_depth_gt = _get(config, "use_lidar_depth_gt", False)
        self.use_depth_gt = _get(config, "use_depth_gt", False)
        assert not (self.use_stereo_depth_gt and self.use_lidar_depth_gt), "only with one depth data supported."
        self.with_depth_gt = self.use_stereo_depth_gt or self.use_lidar_depth_gt or self.use_depth_gt
        if self.dataset == "NYU":
            self.net_3d_decoder = UNet3DNYU(self.n_classes, nn.BatchNorm3d, n_relations=self.n_relations,
                                            feature=self.feature, full_scene_size=self.full_scene_size,
                                            context_prior=self.context_prior, cascade_cls=self.cascade_cls,
                                            infer_mode=self.infer_mode)
        elif self.dataset == "kitti":
            self.net_3d_decoder = UNet3DKitti(self.n_classes, nn.BatchNorm3d, project_scale=self.project_scale,
                                              feature=self.feature, full_scene_size=self.full_scene_size,
                                              context_prior=self.context_prior, cascade_cls=self.cascade_cls,
                                              occluded_cls=self.occluded_cls, infer_mode=self.infer_mode)
        self.net_rgb = UNet2D.build(out_feature=self.feature_2d_oc, use_decoder=True,
                                    backbone_2d_name=config.backbone_2d_name,
                                    return_up_feats=config.return_up_feats)
        self.save_hyperparameters()
        # counted on the device by test_step / validation_step; no state_dict entries (OccDepth.py:131-133)
        self.train_metrics = SSCMetrics(self.n_classes)
        self.val_metrics = SSCMetrics(self.n_classes)
        self.test_metrics = SSCMetrics(self.n_classes)
        self.init_2d_to_3d_trans(config)
        if self.dataset not in ("kitti", "NYU"):
            raise NotImplementedError(self.dataset)

    def init_2d_to_3d_trans(self, config):
        print("INFO: Selected 2d->3d transformation method: {}".format(self.trans_2d_to_3d))
        if self.trans_2d_to_3d in ("flosp", "flosp_depth"):
            self.scale_2ds = [1, 2, 4, 8]
            self.projects = nn.ModuleDict({
                str(s): SFA(config.full_scene_size, project_scale=self.project_scale, dataset=self.dataset)
                for s in self.scale_2ds})
            if self.trans_2d_to_3d == "flosp_depth":
                from .flosp_depth.flosp_depth import FlospDepth, flosp_depth_conf_map
                self.flosp_depth_conf = flosp_depth_conf_map[self.dataset]
                self.flosp_depth_conf.update({
                    "scene_size": config.full_scene_size,
                    "project_scale": config.project_scale,
                    "output_channels": config.feature,
                    "depth_net_conf": dict(in_channels=config.feature,
                                           mid_channels=self.flosp_depth_conf["depth_net_conf"]["mid_channels"]),
                    "return_depth": self.with_depth_gt,
                    "infer_mode": self.infer_mode,
                })
                self.flosp_depth = FlospDepth(**self.flosp_depth_conf)
                if self.with_depth_gt:                                  # DepthClsLoss (OccDepth.py:200-204)
                    self.depth_downsample_factor = self.flosp_depth_conf["downsample_factor"]
                    self.depth_d_bound = list(self.flosp_depth_conf["d_bound"])
        else:
            raise NotImplementedError(f"{self.trans_2d_to_3d} is not supported yet.")

    # ------------------------------------------------------------------------------------------
    def _build(self, B, V, H, W, N, P, dev, batch, classes=None, capture=True, depth_items=False):
        """the launch plan of one batch shape; classes: None (the forward's outputs) or ("classes", lut, *options): the
        plan of predict_classes, whose decoder ends in the uint16 class map (`out` is then that tensor).  Options:
        "conf" -- `out` is uint16 [2, B, X, Y, Z], the map then the float16 bits of its confidence; "probs" -- `out`
        is uint16 [(1 + C) * B, X, Y, Z], the map then the float16 bits of every class's probability
        (modules.split_probs); "root" -- see below.  capture=False: no CUDA graph (and no warm-up run), whatever OCCDEPTH_CUDA_GRAPH says.
        depth_items: NYU's virtual view reads one depth map per batch item (a [B, dh, dw] buffer; predict_frames of
        independent frames) instead of item 0's for the whole batch, as the reference's tensor batches do"""
        slab = self.__dict__.get("slab_ctx")
        plan = Plan(dev, slab=slab, precision=self.precision)
        ps = self.project_scale
        S = [int(s) // ps for s in self.full_scene_size]
        n_lo = 0
        window = None
        plan.x_range = None
        if slab is not None:
            # one frame, X-slab partition: this rank lifts and decodes planes [x_lo, x_hi) of the voxel grid; the
            # 2D network is replicated (its receptive field is global: SE pooling) -- SURVEY.md section 8e.  Both
            # datasets' voxel orders are X-major, so the slab is one contiguous range of projected_pix / fov_mask.
            if B != 1:
                raise NotImplementedError("slab partition: one frame per forward (batch size 1), got %d" % B)
            if self.dataset == "NYU" and self.trans_2d_to_3d == "flosp_depth":
                raise NotImplementedError("slab partition: NYU with the FlospDepth prior is not built (no shipped "
                                          "configuration uses it)")
            # boundaries on multiples of 2^stages: the UNet's two Downsamples, plus the CRP mega-context conv
            stages = 2 + (1 if self.net_3d_decoder.context_prior else 0)
            x_lo, x_hi = slab.partition(S[0], stages)
            n_lo, N = x_lo * S[1] * S[2], (x_hi - x_lo) * S[1] * S[2]
            window = (x_lo, x_hi - x_lo)
            plan.x_range = (x_lo * ps, x_hi * ps)     # this rank's planes of the full-resolution outputs
            S = [x_hi - x_lo, S[1], S[2]]
        virtual = V == 1 and "gt_depth" in batch                          # process_rgbs, OccDepth.py:221-229
        VL = 2 if virtual else V                                           # views seen by the lift
        view_sel = self.slab_view(V, virtual)
        view_shard = view_sel is not None
        img = plan.alloc(B * (1 if view_shard else V), 1, H, W, 3)
        Cf = self.feature_2d_oc
        assert Cf == self.feature, "feature_2d_oc must equal feature (the lift feeds the 3D net directly)"
        if Cf % 4 != 0 or not 0 < Cf <= 256:
            raise NotImplementedError("OccDepth: feature must be a multiple of 4 between 4 and 256 (got %d)" % Cf)
        # every 2-D feature map the lift reads has channel stride Cp; its pad channels [Cf, Cp) are zero (CL.alloc
        # zero-fills, convolutions and the virtual-view kernel write zeros there), so the lift runs over Cp channels
        # and writes zeros into the pad channels of x3d (DESIGN.md section 3)
        Cp = _round_up(Cf, 8)
        scales = [int(s) for s in self.project_res]
        views = {}
        outs = {}
        if virtual:
            # view-major buffers [2, B, h, w, Cp]: the 2D net writes view 0, the virtual-view kernel view 1
            for s in scales:
                h_s, w_s = feature_hw(H, W, s)
                vb = torch.zeros(2, B, h_s, w_s, Cp, dtype=plan.dtype, device=dev)
                views[s] = vb
                outs["1_%d" % s] = CL(vb[0].unsqueeze(1), Cf)
        gathered = None
        if view_shard:
            R2 = slab.world // 2
            hw = [feature_hw(H, W, s) for s in scales]
            offs, P_tot = [], 0
            for (h_s, w_s) in hw:
                offs.append(P_tot)
                P_tot += h_s * w_s
            slice_len = -(-P_tot // R2)
            P_pad = slice_len * R2
            packed = torch.zeros(P_pad, Cp, dtype=plan.dtype, device=dev)       # this rank's view, all scales
            gathered = torch.zeros(2, P_pad, Cp, dtype=plan.dtype, device=dev)  # both views after the all-gather
            for s, (h_s, w_s), o in zip(scales, hw, offs):
                outs["1_%d" % s] = CL(packed[o:o + h_s * w_s].view(1, 1, h_s, w_s, Cp), Cf)
        x_rgb = self.net_rgb.emit(plan, img, outs)                          # {"1_s": CL [B*V,1,h,w,Cf]}
        if view_shard:
            sl = slab.rank % R2
            plan.add(slab.all_gather_op(packed[sl * slice_len:(sl + 1) * slice_len],
                                        gathered.view(2 * R2, slice_len, Cp)))
            for s, (h_s, w_s), o in zip(scales, hw, offs):
                views[s] = gathered[:, o:o + h_s * w_s].view(2, 1, h_s, w_s, Cp)   # [view][B=1][h][w][Cp]
        depth0 = None
        if virtual:
            L = _lib.lib()
            gd = batch["gt_depth"]
            dh, dw = gd.shape[2], gd.shape[3]
            depth0 = torch.zeros(((B,) if depth_items else ()) + (dh, dw), dtype=torch.float32, device=dev)
            bf = float(batch["virtual_bf"][0])
            for s in scales:
                vb = views[s]
                _, _, h_s, w_s, _ = vb.shape
                if depth_items:
                    plan.add(FnOp(lambda st, vb=vb, h_s=h_s, w_s=w_s, s=s: L.occd_virtual_view_items_fwd(
                        vb[0].data_ptr(), vb[1].data_ptr(), depth0.data_ptr(), plan.lib_dtype, B, h_s, w_s, Cf, Cp,
                        Cp, dh, dw, bf / s, dh * dw, st), "virtual_view_1_%d" % s, keep=(vb, depth0)))
                    continue
                plan.add(FnOp(lambda st, vb=vb, h_s=h_s, w_s=w_s, s=s: L.occd_virtual_view_fwd(
                    vb[0].data_ptr(), vb[1].data_ptr(), depth0.data_ptr(), plan.lib_dtype, B, h_s, w_s, Cf, Cp, Cp,
                    dh, dw, bf / s, st), "virtual_view_1_%d" % s, keep=(vb, depth0)))
        pix = torch.zeros(B, VL, N, P, 2, dtype=torch.int64, device=dev)
        fov = torch.zeros(B, VL, N, P, dtype=torch.bool, device=dev)
        x3d = plan.alloc(B, S[0], S[1], S[2], self.feature)
        prior = None
        if self.trans_2d_to_3d == "flosp_depth":
            n_cams = 1 if self.dataset == "NYU" else V                      # OccDepth.py:303-305
            x_depth = x_rgb
            if view_shard:
                # DepthNet runs whole on every rank, over both views' 1_8 maps: after the all-gather they are views
                # of `gathered` with a view stride of P_pad * Cp; one copy per view makes them a dense [2,1,h,w,Cp]
                L = _lib.lib()
                g8 = views[8]
                _, _, h8, w8, _ = g8.shape
                dense = plan.alloc(2, 1, h8, w8, Cf)
                for v in range(2):
                    plan.add(FnOp(lambda st, v=v: L.occd_copy_channels(
                        g8[v].data_ptr(), dense.buf[v].data_ptr(), plan.lib_dtype, h8 * w8, Cp, Cp, 0, Cp, 0, st),
                        "depthnet.gather_views", keep=(gathered, dense)))
                x_depth = {"1_8": dense}
            prior = self.flosp_depth.emit(plan, x_depth, batch, B, V, n_cams, window=window)  # fp32 [B, X*Y*Z]
            plan.flosp_state = self.flosp_depth.plan_state()
        for b in range(B):
            feats = []
            for s in scales:
                if virtual or view_shard:
                    feats.append(views[s][:, b])                            # [2, h, w, Cp], strided views
                else:
                    f = x_rgb["1_%d" % s]
                    assert f.coff == 0 and f.cstride == Cp
                    feats.append(f.buf[b * V:(b + 1) * V, 0])               # [V, h, w, Cp] contiguous view
            out_b = CL(x3d.buf[b:b + 1], x3d.C, 0, x3d.d0, x3d.dlen)
            pr = prior[b] if prior is not None else None
            plan.add(FnOp(lambda st, feats=feats, pb=pix[b], fb=fov[b], ob=out_b, pr=pr:
                          (lift_multiscale(feats, scales, pb, fb, ob, self.dataset,
                                           [S[0] * ps, S[1] * ps, S[2] * ps], ps,
                                           prior=pr, scale_const=100.0, stream=st), 0)[1],
                          "sfa_lift", keep=(feats, pix, fov, out_b)))
        if classes is None:
            out = self.net_3d_decoder.emit(plan, x3d)
        else:
            conf, probs = "conf" in classes[2:], "probs" in classes[2:]
            out = self.net_3d_decoder.emit(plan, x3d, classes=True, lut=classes[1], confidence=conf,
                                           probabilities=probs)
            if "root" in classes[2:]:
                # predict_frame(slab_output="root"): rank 0 gathers the ranks' slabs into the whole map (and its
                # confidence: a second gather of the same shape; or its probabilities: the map and the C probability
                # planes, 1 + C items of one gather), which is then this plan's output there; the other ranks' plans
                # output nothing
                bounds = [(lo * ps, hi * ps) for lo, hi in slab.bounds]       # every rank's plan.x_range
                parts = [out[0], out[1]] if conf else [out]
                whole = None
                if slab.rank == 0:
                    lead = (2, 1) if conf else (out.shape[0],) if probs else (1,)
                    whole = torch.empty(lead + (bounds[-1][1],) + tuple(out.shape[-2:]), dtype=out.dtype, device=dev)
                for k, part in enumerate(parts):
                    plan.add(slab.gather_root_op(part, None if whole is None else (whole[k] if conf else whole),
                                                 bounds))
                out = whole
        if capture and os.environ.get("OCCDEPTH_CUDA_GRAPH", "1") == "1":
            try:
                plan.capture()
            except Exception as e:  # noqa: BLE001 -- same kernels either way; only the launch mechanism differs
                print("WARNING: CUDA graph capture failed (%r); launching kernels individually" % (e,))
                plan.graph = None
        return plan, img, pix, fov, out, depth0, n_lo, view_sel

    def forward(self, batch):
        return self._run(batch, None)

    def predict_classes(self, batch, inv_map=None, confidence=False, probabilities=False):
        """uint16 class per voxel [B, X, Y, Z]: bit for bit `class_map(self(batch)["ssc_logit"], inv_map)`, but the
        classifier's epilogue writes the map, so no logits (and none of the forward's other outputs) are stored,
        converted or copied.  inv_map: one label id per class (at most 64), the submission writer's remap.  Its plan is
        cached apart from the forward's (alternating both rebuilds neither); under enable_slab_parallel this rank's
        X-slab.  confidence=True: returns (map, conf), conf float16 [B, X, Y, Z] each voxel's top-class softmax
        probability, max softmax(ssc_logit), computed by the same epilogue in fp32 and rounded once (NaN where a logit
        is NaN or +inf; inv_map does not touch it).  probabilities=True: returns (map, probs), probs float16
        [B, C, X, Y, Z] every class's softmax probability, softmax(ssc_logit, dim=1), from the same epilogue: exp(l - m)
        / s in fp32 with the confidence's m and s, rounded once (NaN in every class where a logit is NaN or +inf; the
        probability at the map's class is the confidence, bit for bit; inv_map remaps the map only).  The map is the
        same either way."""
        _check_class_request("predict_classes", True, confidence, probabilities)
        return self._run(batch, self._class_key(inv_map, confidence, probabilities=probabilities))

    def _class_key(self, inv_map, confidence=False, root=False, probabilities=False):
        """the `classes` argument of _build (and part of the class-map plan's cache key)"""
        return (("classes", self._class_lut(inv_map)) + (("conf",) if confidence else ())
                + (("probs",) if probabilities else ()) + (("root",) if root else ()))

    def _class_lut(self, inv_map):
        if inv_map is None:
            return None
        import numpy as np
        lut = tuple(int(v) for v in np.asarray(inv_map).astype(np.int64).reshape(-1))
        if len(lut) != self.n_classes:
            raise ValueError("OccDepth.predict_classes: inv_map must hold one label id per class")
        return lut

    def slab_view(self, V, virtual=False):
        """the one view of a V-view frame this rank's plan stages under enable_slab_parallel, or None (every view).
        Over an even number of ranks a stereo frame's 2D network is sharded BY VIEW (its receptive field is global
        inside a view -- SE pooling -- but the two views are independent, process_rgbs OccDepth.py:208-219): ranks
        [0, R/2) run view 0, ranks [R/2, R) view 1, and one all-gather hands every rank both views' maps.  `virtual`:
        the frame's second view is NYU's virtual one, computed from the first."""
        slab = self.__dict__.get("slab_ctx")
        if (slab is None or V != 2 or virtual or slab.world % 2
                or os.environ.get("OCCDEPTH_SLAB_VIEW_SHARD", "1") != "1"):
            return None
        return slab.rank // (slab.world // 2)

    def _plan_key(self, B, V, H, W, N, P, dev, virtual, virtual_bf):
        """cache key of the launch plan of one batch shape (shared by tensor batches and camera frames)"""
        slab = self.__dict__.get("slab_ctx")
        return (B, V, H, W, N, P, str(dev), virtual, virtual_bf if virtual else 0.0,
                None if slab is None else (slab.rank, slab.world), self.precision, self.param_stamp())

    def _run(self, batch, classes):
        img = batch["img"]
        if not img.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("OccDepth.forward: occdepth_b200 needs a CUDA (sm_90a) device")
            img = img.cuda(non_blocking=True)          # the reference moves the batch in forward too (:345)
        self._check_mode(img)
        dev = img.device
        if next(self.parameters()).device != dev:
            raise RuntimeError("OccDepth.forward: model and batch are on different devices")
        B, V, _, H, W = img.shape
        ps = self.project_scale
        pp = batch["projected_pix_{}".format(ps)]
        fm = batch["fov_mask_{}".format(ps)]
        N, P = pp[0].shape[1], pp[0].shape[2]
        virtual = V == 1 and "gt_depth" in batch
        key = self._plan_key(B, V, H, W, N, P, dev, virtual, float(batch["virtual_bf"][0]) if virtual else 0.0)
        stage = lambda ent: self._stage(ent, batch, img, pp, fm, dev)    # noqa: E731
        with torch.cuda.device(dev):           # launches, tensor maps and function attributes follow the tensors
            if classes is not None:
                return self._classes_on(batch, key + classes, B, V, H, W, N, P, dev, classes, stage)
            return self._forward_on(batch, key, B, V, H, W, N, P, dev, stage)

    def prepare(self, batch):
        """build and cache the launch plan (weight snapshot, buffers, tensor maps, CUDA graph) for this batch's
        shapes without running it: the first forward() then costs what every later one does.  No collective is
        executed, so a multi-rank caller can agree on success before any rank starts a halo exchange."""
        self.__dict__["_build_only"] = True
        try:
            self.forward(batch)
        finally:
            self.__dict__.pop("_build_only", None)
        return self

    def _forward_on(self, batch, key, B, V, H, W, N, P, dev, stage, n=None, depth_items=False):
        """batch: what _build reads (shapes, the virtual view, vox_origin); stage(ent) fills the plan's inputs.
        n: items [0, n) of every output (a short list of camera frames through a B-frame plan)"""
        ent = self._plans().get(key)
        if ent is None:
            self._plans().clear()              # weights changed / new shape: drop the stale snapshot
            with torch.no_grad():
                ent = self._build(B, V, H, W, N, P, dev, batch, depth_items=depth_items)
            self._plans()[key] = ent
        if self.__dict__.get("_build_only"):
            return None
        stage(ent)
        ent[0].run()
        res = self._outputs(ent)
        if n is not None and n != B:
            res = {k: (v[:n] if isinstance(v, torch.Tensor) and v.dim() and v.shape[0] == B else v)
                   for k, v in res.items()}
        return res

    def _classes_on(self, batch, key, B, V, H, W, N, P, dev, classes, stage, n=None, depth_items=False):
        """n: return items [0, n) of the class map (a short list of camera frames through a B-frame plan)"""
        cache = self._class_plans()
        ent = cache.get(key)
        if ent is None:
            cache.clear()                      # one class-map plan: weights, shapes or inv_map changed
            with torch.no_grad():
                ent = self._build(B, V, H, W, N, P, dev, batch, classes=classes, depth_items=depth_items)
            cache[key] = ent
        if self.__dict__.get("_build_only"):
            return None
        stage(ent)
        ent[0].run()
        if ent[4] is None:                     # slab_output="root" on a rank other than 0
            return None
        n = B if n is None else n
        if "conf" in classes[2:]:              # uint16 [2, ...]: the map, then the confidence's float16 bits
            return ent[4][0, :n].clone(), ent[4][1, :n].clone().view(torch.float16)
        if "probs" in classes[2:]:             # the map, then every class's float16 probability
            cmap, probs = split_probs(ent[4], B)
            return cmap[:n].clone(), probs[:n].clone()
        return ent[4][:n].clone()              # the map lives in a plan-owned static buffer

    def _stage(self, ent, batch, img, pp, fm, dev):
        """copy this batch's inputs into the static input buffers of plan entry `ent`"""
        plan, img_cl, pix, fov, out, depth0, n_lo, view_sel = ent
        plan.calib_mark = None                 # the index buffers no longer hold camera frames' calibrations
        B, V, _, H, W = img.shape
        CL.from_planar(img.reshape(B * V, 3, H, W) if view_sel is None else img[:, view_sel].reshape(B, 3, H, W),
                       out=img_cl)
        if depth0 is not None:
            depth0.copy_(batch["gt_depth"][0, 0], non_blocking=True)
        nl = pix.shape[2]
        for b in range(B):
            pix[b].copy_(pp[b][:, n_lo:n_lo + nl], non_blocking=True)
            fov[b].copy_(fm[b][:, n_lo:n_lo + nl], non_blocking=True)
        if self.trans_2d_to_3d == "flosp_depth":
            self.flosp_depth.stage_inputs(batch, dev, plan.flosp_state)

    # ---- camera frames: uint8 images and calibration in, the datasets' pre-processing on the device -------------
    def predict_frame(self, frame, classes=True, inv_map=None, slab_output=None, confidence=False,
                      probabilities=False):
        """One camera frame -> the class map (classes=True: uint16 [1, X, Y, Z], `inv_map`, `confidence` and
        `probabilities` as in
        predict_classes) or the forward's output dict (classes=False), through the same cached plan a tensor batch of the same shapes
        uses.  Only the staging differs: the datasets' pre-processing (eval split, no augmentation) runs on the device
        and writes the plan's input buffers -- the images through `occd_stage_rgb_u8_cl`, the indices through
        `occd_vox2pix_fwd`, NYU's depth map through `occd_depth_u16_to_f32`.

        frame (host arrays or tensors; the images and depth map may already be on the device):
          "img": uint8 RGB (V, H0, W0, 3), or (H0, W0, 3) for one view: the decoded camera images, cropped to
                 `img_hw` on the device (kitti_dataset.py:376-402)
          KITTI: "cam_k" (V, 3, 3) and "T_velo_2_cam" (V, 4, 4) (kitti_dataset.py:196-290)
          NYU:   "cam_pose" (4, 4), "vox_origin" (3,), "cam_k" (3, 3) (default: the dataset's), "depth": the uint16
                 depth PNG (H, W) when the model runs the virtual right view (nyu_dataset.py:116-200)
          optional geometry, fixed per dataset: "img_hw" (KITTI (370, 1220), NYU (480, 640)), "vox_origin" (KITTI
          (0, -25.6, -2)), "voxel_size" (KITTI 0.2 * project_scale, NYU 0.08), "scene_size", "pattern_id" (0)
          camera formats (`occd_stage_camera_u8_cl`; bit for bit what OpenCV makes of the frame on the host):
          "pixel_format": "rgb" (default), "bgr", or "nv12" -- then "img" is uint8 (V, H0 * 3 / 2, W0), OpenCV's
                 NV12 layout (cv2.COLOR_YUV2RGB_NV12), H0 and W0 even
          "rect_maps": float32 (V, 2, img_h, img_w), each view's cv2.initUndistortRectifyMap x and y maps: the images
                 are rectified as cv2.remap(INTER_LINEAR, BORDER_CONSTANT) does, and "cam_k" is the rectified
                 camera's.  Read in place on the device; host maps are copied every call.  NYU's depth map is not
                 remapped: it must already be in the rectified camera's frame.
          Neither changes the plan.
        The indices are recomputed only when the calibration differs from what the plan's index buffers hold (a KITTI
        sequence keeps one); NYU poses change every frame.  One frame per call.

        Under enable_slab_parallel every rank is handed the same frame and `slab_output` says which result it wants:
          "slab": this rank's X-slab, as predict_classes returns it (classes=False: the forward's per-rank dict);
          "root": (classes=True only) rank 0 returns the whole [1, X, Y, Z] map (with `confidence` the whole (map,
                  conf), with `probabilities` the whole (map, probs)), bit for bit the unpartitioned one, gathered from
                  the ranks' slabs; the other ranks return None.
        Each rank stages its own view under view sharding (else every view), the whole depth map, and the indices of
        its X-slab only (`occd_vox2pix_range_fwd`).  Without slab_output the partition is refused; without the
        partition slab_output must be None."""
        if confidence and not classes:
            raise ValueError("OccDepth.predict_frame: confidence=True is the class map's confidence (classes=True)")
        _check_class_request("predict_frame", classes, confidence, probabilities)
        return self._run_frame(self._frame_checked(frame, slab_output, classes), classes, inv_map, slab_output,
                               confidence, probabilities)

    def _frame_checked(self, frame, slab_output=None, classes=True):
        """the refusals of the camera route, then `_frame_inputs`"""
        if slab_output not in (None, "slab", "root"):
            raise ValueError("OccDepth.predict_frame: slab_output must be None, 'slab' or 'root', got %r"
                             % (slab_output,))
        if self.__dict__.get("slab_ctx") is None:
            if slab_output is not None:
                raise ValueError("OccDepth.predict_frame: slab_output=%r needs enable_slab_parallel" % (slab_output,))
        elif slab_output is None:
            raise NotImplementedError("OccDepth.predict_frame: under enable_slab_parallel a camera frame needs "
                                      "slab_output='slab' (every rank's X-slab) or 'root' (the whole map on rank 0)")
        if slab_output == "root" and not classes:
            raise ValueError("OccDepth.predict_frame: slab_output='root' gathers the class map (classes=True); the "
                             "logits stay on their ranks (slab_output='slab')")
        if self.infer_mode and self.trans_2d_to_3d == "flosp_depth":
            raise NotImplementedError("OccDepth.predict_frame: infer_mode with flosp_depth takes the caller's sampling "
                                      "grids, not camera matrices; use forward / predict_classes with a tensor batch")
        dev = next(self.parameters()).device
        self._check_mode(torch.empty(0, device=dev))
        return self._frame_inputs(frame, dev)

    def _run_frame(self, f, classes, inv_map, slab_output=None, confidence=False, probabilities=False):
        dev = f["imgs"].device
        key = self._plan_key(1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["virtual"], f["virtual_bf"])
        stage = lambda ent: self._stage_frame(ent, f)     # noqa: E731
        with torch.cuda.device(dev):
            if classes:
                cls = self._class_key(inv_map, confidence, slab_output == "root", probabilities)
                return self._classes_on(f["batch"], key + cls, 1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, cls,
                                        stage)
            return self._forward_on(f["batch"], key, 1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, stage)

    def _frame_inputs(self, frame, dev):
        """host side of predict_frame: the views' poses, the geometry, the stand-in batch _build and FlospDepth read"""
        import numpy as np
        from .. import data as D
        img = frame["img"]
        if not isinstance(img, torch.Tensor):
            img = torch.from_numpy(np.ascontiguousarray(img))
        fmt = frame.get("pixel_format", "rgb")
        if fmt not in _lib.PIXEL_FORMATS:
            raise ValueError("OccDepth.predict_frame: frame['pixel_format'] must be 'rgb', 'bgr' or 'nv12', got %r"
                             % (fmt,))
        if fmt == "nv12":
            if img.dim() == 2:
                img = img.unsqueeze(0)
            # 3 * H / 2 rows: a multiple of 3 exactly when H is even
            if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[1] % 3 or img.shape[2] % 2:
                raise ValueError("OccDepth.predict_frame: an NV12 frame['img'] must be uint8 (V, H * 3 / 2, W), "
                                 "OpenCV's NV12 layout, with H and W even")
            if img.stride(2) != 1:
                img = img.contiguous()
        else:
            if img.dim() == 5:
                if img.shape[0] != 1:
                    raise NotImplementedError("OccDepth.predict_frame: one frame per call (batch size %d)"
                                              % img.shape[0])
                img = img[0]
            if img.dim() == 3:
                img = img.unsqueeze(0)
            if img.dtype != torch.uint8 or img.dim() != 4 or img.shape[3] != 3:
                raise ValueError("OccDepth.predict_frame: frame['img'] must be uint8 RGB (V, H, W, 3)")
            if img.stride(3) != 1 or img.stride(2) != 3:
                img = img.contiguous()
        img = img.to(dev, non_blocking=True)
        V = int(img.shape[0])
        nyu = self.dataset == "NYU"
        H, W = (int(v) for v in frame.get("img_hw", (480, 640) if nyu else (370, 1220)))
        maps = frame.get("rect_maps")
        if maps is not None:
            if not isinstance(maps, torch.Tensor):
                maps = torch.from_numpy(np.ascontiguousarray(maps))
            if maps.dtype != torch.float32 or tuple(maps.shape) != (V, 2, H, W):
                raise ValueError("OccDepth.predict_frame: frame['rect_maps'] must be float32 (%d, 2, %d, %d): each "
                                 "view's source x and y per pixel of the %d x %d crop" % (V, H, W, H, W))
            maps = maps.to(dev, non_blocking=True)
            if not maps[0].is_contiguous():
                maps = maps.contiguous()
        g = dict(voxel_size=frame.get("voxel_size", 0.08 if nyu else 0.2 * self.project_scale),
                 scene_size=tuple(frame.get("scene_size", (4.8, 4.8, 2.88) if nyu else (51.2, 51.2, 6.4))),
                 pattern_id=int(frame.get("pattern_id", 0)))
        depth, bf = None, 0.0
        if nyu:                                                   # nyu_dataset.py:126-190, collate.py:31-41
            if V != 1:
                raise ValueError("OccDepth.predict_frame: an NYU frame holds one image")
            cam_k = np.asarray(frame.get("cam_k", [[518.8579, 0, 320], [0, 518.8579, 240], [0, 0, 1]]))
            cam_k = cam_k.reshape(3, 3)
            vox_origin = np.asarray(frame["vox_origin"])
            T_world_2_cam = np.linalg.inv(np.asarray(frame["cam_pose"]))
            poses = [(T_world_2_cam, cam_k)]
            depth = frame.get("depth")
            batch = {"cam_k": [torch.from_numpy(np.array([cam_k])).double()],
                     "T_velo_2_cam": [torch.from_numpy(T_world_2_cam[np.newaxis, ...]).float()],
                     "ida_mats": [torch.eye(4).unsqueeze(0)], "vox_origin": torch.from_numpy(vox_origin[None]).double()}
            if depth is not None:
                virtual_baseline = 0.1
                T_cam0_2_cam1 = np.array([[1, 0, 0, -virtual_baseline], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
                poses.append((T_cam0_2_cam1 @ T_world_2_cam, cam_k))
                bf = float(np.array(virtual_baseline * 518.8579))
                if not isinstance(depth, torch.Tensor):
                    depth = torch.from_numpy(np.ascontiguousarray(depth))
                if depth.dtype != torch.uint16 or depth.dim() != 2:
                    raise ValueError("OccDepth.predict_frame: frame['depth'] must be the uint16 depth PNG (H, W)")
                depth = depth.contiguous().to(dev, non_blocking=True)
                batch.update(gt_depth=torch.empty((1, 1) + tuple(depth.shape), device="meta"), virtual_bf=[bf])
            calib = None                                          # a new pose every frame
        else:                                                     # kitti_dataset.py:196-290, collate.py:26-28
            cam_k = np.asarray(frame["cam_k"])
            T = np.asarray(frame["T_velo_2_cam"])
            if cam_k.shape != (V, 3, 3) or T.shape != (V, 4, 4):
                raise ValueError("OccDepth.predict_frame: a KITTI frame of %d images needs cam_k (%d, 3, 3) and "
                                 "T_velo_2_cam (%d, 4, 4)" % (V, V, V))
            vox_origin = np.asarray(frame.get("vox_origin", np.array([0, -25.6, -2])))
            poses = [(T[v], cam_k[v]) for v in range(V)]
            # img_transform((0, 0, W, H), False) is the identity (kitti_dataset.py:380-390)
            batch = {"cam_k": [torch.from_numpy(cam_k).double()], "T_velo_2_cam": [torch.from_numpy(T).float()],
                     "ida_mats": [torch.eye(4).unsqueeze(0).repeat(V, 1, 1)]}
            calib = tuple((a.dtype.str, a.shape, a.tobytes()) for a in (T, cam_k, vox_origin)) + \
                (float(g["voxel_size"]), g["scene_size"], g["pattern_id"], H, W)
        X, Y, Z = (int(v) for v in D.volume_dims(vox_origin, g["voxel_size"], g["scene_size"]))
        S = [int(s) // self.project_scale for s in self.full_scene_size]
        if X * Y * Z != S[0] * S[1] * S[2]:
            raise ValueError("OccDepth.predict_frame: the geometry gives a %dx%dx%d voxel grid, the model lifts into "
                             "%dx%dx%d" % (X, Y, Z, S[0], S[1], S[2]))
        if not 0 <= g["pattern_id"] < len(D.PIXEL_PATTERNS):
            raise IndexError("pattern_id out of range")
        return dict(g, imgs=img, pixel_format=fmt, maps=maps, V=V, H=H, W=W, N=X * Y * Z,
                    P=len(D.PIXEL_PATTERNS[g["pattern_id"]]), poses=poses, vox_origin=vox_origin, depth=depth,
                    virtual=depth is not None, virtual_bf=bf, batch=batch, calib=calib)

    def _stage_frame(self, ent, f, b=0):
        """the device side of predict_frame / predict_frames: stage frame `f` into batch item b of the static input
        buffers of plan entry `ent`.  The item's indices and camera tables are recomputed only when its calibration
        differs from what the item's own buffers hold"""
        from .. import data as D
        plan, img_cl, pix, fov, out, depth0, n_lo, view_sel = ent
        B = pix.shape[0]
        if getattr(plan, "calib_mark", None) is None:
            plan.calib_mark = [None] * B         # per item: the calibration its index buffers hold
        if getattr(plan, "pix_z", None) is None:
            plan.pix_z = torch.empty(B, pix.shape[2], dtype=torch.float64, device=pix.device)   # vox2pix's depths
        imgs = f["imgs"] if view_sel is None else f["imgs"][view_sel:view_sel + 1]
        n_img = imgs.shape[0]
        if f["pixel_format"] == "rgb" and f["maps"] is None:
            D.stage_rgb_u8(imgs, img_cl.buf[b * n_img:(b + 1) * n_img], img_cl.lib_dtype, f["H"], f["W"])
        else:
            maps = f["maps"] if f["maps"] is None or view_sel is None else f["maps"][view_sel:view_sel + 1]
            D.stage_camera_u8(imgs, img_cl.buf[b * n_img:(b + 1) * n_img], img_cl.lib_dtype, f["H"], f["W"],
                              f["pixel_format"], maps)
        if depth0 is not None:
            d = depth0 if depth0.dim() == 2 else depth0[b]
            if tuple(f["depth"].shape) != tuple(d.shape):
                raise ValueError("OccDepth.predict_frame: depth map %r, the plan holds %r"
                                 % (tuple(f["depth"].shape), tuple(d.shape)))
            D.depth_u16_to_f32(f["depth"], d)
        if f["calib"] is not None and f["calib"] == plan.calib_mark[b]:
            return                              # same calibration: the indices and camera tables are in place
        # under the slab partition the index buffers hold this rank's window [n_lo, n_lo + N) of the lift's X-major
        # voxel order: the rank computes that window only, for every pose (NYU's virtual view too)
        window = None if plan.x_range is None else (n_lo, pix.shape[2])
        for v, (E, K) in enumerate(f["poses"]):
            D.vox2pix_into(pix[b, v], fov[b, v], plan.pix_z[b], E, K, f["vox_origin"], f["voxel_size"], f["W"], f["H"],
                           f["scene_size"], f["pattern_id"], voxel_range=window)
        if self.trans_2d_to_3d == "flosp_depth":
            self.flosp_depth.stage_inputs(f["batch"], pix.device, plan.flosp_state, item=b)
        plan.calib_mark[b] = f["calib"]

    # ---- batches of camera frames ----------------------------------------------------------------------------------
    def predict_frames(self, frames, classes=True, inv_map=None, confidence=False, probabilities=False):
        """A list of 1..B camera frames (each what predict_frame takes) through one B-frame plan, B = len(frames): the
        uint16 class maps [n, X, Y, Z] (with `confidence`: (map, conf); with `probabilities`: (map, probs), probs
        float16 [n, C, X, Y, Z]), or with classes=False the forward's output dict
        with a leading n.  Every frame's result is bit for bit predict_frame's of that frame alone.

        The frames must agree on the image count V, the crop `img_hw`, the grid geometry (voxel_size, scene_size,
        pattern_id) and whether there is a depth map; calibration, pose, NYU's vox_origin and the raw image sizes may
        differ (each frame's images are staged by their own launch).  NYU's virtual view reads each frame's own depth
        map (all of the size the plan was built with).  One plan is cached per batch size and request; each batch item
        keeps the calibration its index buffers hold, so a KITTI sequence computes the indices once per item.  Not
        under enable_slab_parallel with more than one frame, nor for NYU with the FlospDepth prior with more than one
        (its grid is rebuilt from item 0's vox_origin)."""
        fs = self._frames_checked(frames, classes, confidence, probabilities=probabilities)
        return self._run_frames(fs, len(fs), classes, inv_map, confidence, probabilities)

    def _frames_checked(self, frames, classes=True, confidence=False, batch=None, inputs=True, probabilities=False):
        """the refusals of predict_frames (host-side, before any frame is moved), then -- with `inputs` -- the frames
        through `_frame_checked`"""
        if isinstance(frames, dict) or not isinstance(frames, (list, tuple)):
            raise TypeError("OccDepth.predict_frames: frames must be a list of frame dicts")
        n = len(frames)
        if n < 1 or (batch is not None and n > batch):
            raise ValueError("OccDepth.predict_frames: %d frames, expected 1 to %s" % (n, "any" if batch is None
                                                                                       else batch))
        if confidence and not classes:
            raise ValueError("OccDepth.predict_frames: confidence=True is the class map's confidence (classes=True)")
        _check_class_request("predict_frames", classes, confidence, probabilities)
        B = n if batch is None else batch
        if self.__dict__.get("slab_ctx") is not None and B > 1:
            raise NotImplementedError("OccDepth.predict_frames: the slab partition runs one frame per forward (batch "
                                      "size 1), got %d" % B)
        if self.infer_mode and self.trans_2d_to_3d == "flosp_depth":
            raise NotImplementedError("OccDepth.predict_frames: infer_mode with flosp_depth takes the caller's sampling "
                                      "grids, not camera matrices; use forward / predict_classes with a tensor batch")
        if self.dataset == "NYU" and self.trans_2d_to_3d == "flosp_depth" and B > 1:
            raise NotImplementedError("OccDepth.predict_frames: NYU with the FlospDepth prior rebuilds its grid from "
                                      "item 0's vox_origin, so it runs one frame per call (no shipped configuration "
                                      "uses it)")
        sig0 = self._frame_signature(frames[0])
        for i, fr in enumerate(frames[1:], 1):
            sig = self._frame_signature(fr)
            for k in sig0:
                if sig[k] != sig0[k]:
                    raise ValueError("OccDepth.predict_frames: frame %d's %s is %r, frame 0's %r (the frames of one "
                                     "call share it)" % (i, k, sig[k], sig0[k]))
        return [self._frame_checked(fr, None, classes) for fr in frames] if inputs else None

    def _frame_signature(self, frame):
        """what the frames of one predict_frames call must share, read on the host with predict_frame's defaults"""
        nyu = self.dataset == "NYU"
        shape = tuple(getattr(frame["img"], "shape", ()))
        if frame.get("pixel_format", "rgb") == "nv12":
            V = 1 if len(shape) == 2 else shape[0] if len(shape) == 3 else None
        else:
            V = 1 if len(shape) == 3 else shape[-4] if len(shape) >= 4 else None
        return {"V": V,
                "img_hw": tuple(int(v) for v in frame.get("img_hw", (480, 640) if nyu else (370, 1220))),
                "voxel_size": float(frame.get("voxel_size", 0.08 if nyu else 0.2 * self.project_scale)),
                "scene_size": tuple(float(v) for v in frame.get("scene_size", (4.8, 4.8, 2.88) if nyu
                                                                 else (51.2, 51.2, 6.4))),
                "pattern_id": int(frame.get("pattern_id", 0)),
                "depth": frame.get("depth") is not None}

    def _run_frames(self, fs, B, classes, inv_map, confidence=False, probabilities=False):
        """frames fs (from _frames_checked) through the B-frame plan, B >= len(fs): the results of items [0, len(fs));
        items [len(fs), B) keep what their buffers hold"""
        f = fs[0]
        dev = f["imgs"].device
        depth_items = f["virtual"] and B > 1
        # only a batch of camera frames with per-item depth maps gets a key of its own: every other plan is the one a
        # tensor batch of the same shapes uses
        key = self._plan_key(B, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["virtual"], f["virtual_bf"]) \
            + (("depth_items",) if depth_items else ())
        stage = lambda ent: [self._stage_frame(ent, f, b) for b, f in enumerate(fs)]     # noqa: E731
        with torch.cuda.device(dev):
            if classes:
                cls = self._class_key(inv_map, confidence, probabilities=probabilities)
                return self._classes_on(f["batch"], key + cls, B, f["V"], f["H"], f["W"], f["N"], f["P"], dev, cls,
                                        stage, n=len(fs), depth_items=depth_items)
            return self._forward_on(f["batch"], key, B, f["V"], f["H"], f["W"], f["N"], f["P"], dev, stage,
                                    n=len(fs), depth_items=depth_items)

    # ---- the occupied-voxel list: what every consumer of a class map builds from it first ----------------------
    def predict_voxels(self, batch_or_frame, inv_map=None, fov_mask=None, capacity=None, voxel_size=None,
                       vox_origin=None, out=None, slab_output=None):
        """`predict_classes` (a tensor batch: it carries "projected_pix_<project_scale>") or `predict_frame` (a camera
        frame), then `voxels.occupied_voxels` of the class map on the same stream -> VoxelList: per frame the counts,
        the class histogram and the rows (flat index, class, voxel centre) of the occupied voxels, inside the FOV
        first, in numpy's order; nothing is read back until the caller asks the list for counts or rows.

        fov_mask: None takes the frame's `fov_mask_1` -- batch["fov_mask_1"] when the batch has it (what
                  generate_output.py saves for the visualisation scripts), and for a camera frame the mask `vox2pix`
                  gives at the output resolution, computed on the device and kept while the calibration stays the same
                  (once for a KITTI sequence).  A per-frame mask of the datasets' shape (V, N, P) stands for its first
                  view's centre pixel, `[0, :, 0]`, as in kitti_vis_pred_batch.py:92-93.  False: no mask.  NYU has no
                  default mask: its `fov_mask_1` follows vox2pix's (x, y, z) voxel order, not the prediction's
                  (x, z, y), and NYU_vis_pred.py keeps one list.
        voxel_size: of the output grid (default 0.2 for KITTI, 0.08 for NYU); vox_origin: added to the centres.
        inv_map, capacity, out: as in predict_classes / occupied_voxels.
        Under enable_slab_parallel (tensor batches, and camera frames with slab_output="slab") the list holds this
        rank's X-slab with the whole grid's flat indices and coordinates: the ranks' in-FOV rows concatenated in rank
        order, then their out-of-FOV rows, are the unpartitioned list.  A camera frame's default mask is then this
        rank's window of it, from `occd_vox2pix_range_fwd`.  slab_output="root": rank 0 lists the gathered whole map
        (the unpartitioned list exactly), the other ranks return None.

        A list of camera frames runs through predict_frames' B-frame plan (B = len(list), the same plan and key) and
        gives one VoxelList with B = n: frame i's counts, histogram and rows bit for bit those of predict_voxels of
        frame i alone.  Each list position keeps its own default mask while its calibration stays the same; an
        explicit fov_mask holds one mask per frame.  The frames are refused as predict_frames refuses them (so a list
        under enable_slab_parallel is), and slab_output must be None."""
        if isinstance(batch_or_frame, (list, tuple)):
            return self._predict_voxels_list(batch_or_frame, inv_map, fov_mask, capacity, voxel_size, vox_origin, out,
                                             slab_output)
        if not isinstance(batch_or_frame, Mapping):
            raise TypeError("OccDepth.predict_voxels: takes a tensor batch, a camera frame dict or a list of camera "
                            "frames, got %s" % type(batch_or_frame).__name__)
        window_mask = None
        if "projected_pix_%d" % self.project_scale in batch_or_frame:
            y = self.predict_classes(batch_or_frame, inv_map)
            x_range = self.slab_x_range()
            if fov_mask is None:
                fov_mask = False if self.dataset == "NYU" else batch_or_frame.get("fov_mask_1", False)
        else:
            f = self._frame_checked(batch_or_frame, slab_output)
            y = self._run_frame(f, True, inv_map, slab_output)
            x_range = self.slab_x_range() if slab_output == "slab" else None
            if fov_mask is None and y is not None:
                if self.dataset == "NYU":
                    fov_mask = False
                else:
                    window_mask = self._frame_fov_mask_1(f, x_range)
        if y is None:                          # prepare(): the plan was built, nothing ran (or "root" off rank 0)
            return None
        return self._list_voxels(y, x_range, fov_mask, capacity, voxel_size, vox_origin, out, window_mask)

    def _predict_voxels_list(self, frames, inv_map, fov_mask, capacity, voxel_size, vox_origin, out, slab_output):
        """predict_voxels of a list of camera frames: the refusals (host-side, before any device work), the B-frame
        plan, then one listing of its n maps"""
        if slab_output is not None:
            raise ValueError("OccDepth.predict_voxels: a list of frames takes no slab_output (the slab partition runs "
                             "one frame per forward)")
        for i, fr in enumerate(frames):
            if not isinstance(fr, Mapping) or "projected_pix_%d" % self.project_scale in fr:
                raise TypeError("OccDepth.predict_voxels: item %d of the list is not a camera frame dict" % i)
        fs = self._frames_checked(frames)
        y = self._run_frames(fs, len(fs), True, inv_map)
        if y is None:                          # prepare(): the plan was built, nothing ran
            return None
        window_mask = None
        if fov_mask is None:
            if self.dataset == "NYU":
                fov_mask = False
            else:
                window_mask = torch.stack([self._frame_fov_mask_1(f, None, b) for b, f in enumerate(fs)])
        return self._list_voxels(y, None, fov_mask, capacity, voxel_size, vox_origin, out, window_mask)

    def _list_voxels(self, y, x_range, fov_mask, capacity, voxel_size, vox_origin, out, window_mask=None):
        """the list of class map `y` [B, Xl, Y, Z]: the whole grid, or planes x_range = [lo, hi) of it.  fov_mask holds
        the whole grid per frame; window_mask ([B, ...] on the device) only y's planes of it"""
        from ..voxels import occupied_voxels
        B, _, Y, Z = y.shape
        lo, hi = (0, y.shape[1]) if x_range is None else x_range
        n_full = int(self.full_scene_size[0]) * Y * Z
        mask = None
        if window_mask is not None:
            mask = window_mask.view(B, -1)
        elif fov_mask is not None and fov_mask is not False:
            frames = [fov_mask] if getattr(fov_mask, "ndim", 0) == 1 else list(fov_mask)
            rows = []
            for m in frames:
                m = torch.as_tensor(m)
                if m.dim() == 3:               # the datasets' (V, N, P)
                    m = m[0, :, 0]
                if m.numel() != n_full:
                    raise ValueError("OccDepth.predict_voxels: a frame's fov_mask holds %d values, the output grid %d "
                                     "voxels" % (m.numel(), n_full))
                rows.append(m.reshape(-1)[lo * Y * Z:hi * Y * Z].to(y.device, non_blocking=True))
            if len(rows) != B:
                raise ValueError("OccDepth.predict_voxels: %d masks for %d frames" % (len(rows), B))
            mask = torch.stack(rows)
        if voxel_size is None:
            voxel_size = 0.08 if self.dataset == "NYU" else 0.2
        return occupied_voxels(y, mask, voxel_size=voxel_size, vox_origin=vox_origin, capacity=capacity,
                               index0=lo * Y * Z, out=out)

    def _frame_fov_mask_1(self, f, x_range=None, item=None):
        """bool [N] on the device: the first view's `fov_mask_1` of camera frame `f`, i.e. vox2pix at the output
        resolution (kitti_dataset.py:259-273 with scale_3d = 1), centre pixel only; x_range = [lo, hi): only those X
        planes of it.  Kept with the calibration and window it was computed from: one mask for single frames, one per
        list position `item` for lists of frames.  Computed without the pixel indices (`occd_vox2pix_fwd` with no
        pix), as the model-file runtime computes it."""
        import numpy as np
        from .. import data as D
        if item is None:
            held = self.__dict__.get("_fov_mask_1")
        else:
            held = self.__dict__.setdefault("_fov_masks_1", {}).get(item)
        key = (f["calib"], x_range)
        if f["calib"] is not None and held is not None and held[0] == key and held[1].device == f["imgs"].device:
            return held[1]
        voxel = f["voxel_size"] / self.project_scale
        n1 = int(np.prod(D.volume_dims(f["vox_origin"], voxel, f["scene_size"])))
        if n1 != int(np.prod([int(s) for s in self.full_scene_size])):
            raise ValueError("OccDepth.predict_voxels: the geometry gives %d voxels at the output resolution, the model "
                             "predicts %d" % (n1, int(np.prod([int(s) for s in self.full_scene_size]))))
        window, n = None, n1
        if x_range is not None:
            plane = n1 // int(self.full_scene_size[0])
            window = (x_range[0] * plane, (x_range[1] - x_range[0]) * plane)
            n = window[1]
        dev = f["imgs"].device
        E, K = f["poses"][0]
        with torch.cuda.device(dev):
            fov = torch.empty(n, 1, dtype=torch.bool, device=dev)
            D.vox2pix_into(None, fov, None, E, K, f["vox_origin"], voxel, f["W"], f["H"], f["scene_size"], 0,
                           voxel_range=window)
        mask = fov.view(-1)
        if item is None:
            self.__dict__["_fov_mask_1"] = (key, mask)
        else:
            self.__dict__["_fov_masks_1"][item] = (key, mask)
        return mask

    def _outputs(self, ent):
        """the forward's output dict from plan entry `ent` after it ran (under the slab partition: this rank's
        X-slab of every 3-D tensor, its columns of P_logits, and the whole depth_pred)"""
        plan, out = ent[0], ent[4]
        res = _to_planar(out, False)
        # tensors written directly by kernels live in plan-owned static buffers: hand out copies
        res = {k: (v.clone() if isinstance(out[k], torch.Tensor) else v) for k, v in res.items()}
        if self.with_depth_gt and self.trans_2d_to_3d == "flosp_depth":
            res["depth_pred"] = self.flosp_depth.depth_prob(plan.flosp_state).clone()   # OccDepth.py:374-375
        return res

    @staticmethod
    def class_map(ssc_logit, inv_map=None, confidence=False, probabilities=False):
        """uint16 class per voxel from the fp32 logits [B, C, X, Y, Z] on the GPU -- what the reference's callers
        compute on the host after copying all logits back (`np.argmax(torch.softmax(pred["ssc_logit"], 1).cpu(),
        1).astype(np.uint16)`, scripts/generate_output.py:94-97; eval.py does the same).  168 MB of logits shrink to
        a 4 MB map before the device->host read.  `inv_map` (int array of C label ids, io_data.get_inv_map) applies the
        submission writer's remap `inv_map[y_pred].astype(np.uint16)` (generate_kitti_submission.py:79) in the same
        launch.  confidence=True: returns (map, conf), conf float16 [B, X, Y, Z] the top class's softmax probability
        (occd_argmax_classes_conf; NaN where a logit is NaN or +inf; the remap does not touch it).
        probabilities=True: returns (map, probs), probs float16 [B, C, X, Y, Z] every class's softmax probability
        (occd_class_probs: bit for bit what predict_classes(probabilities=True) writes from the same logits)."""
        from .. import _lib
        _check_class_request("class_map", True, confidence, probabilities)
        if not (ssc_logit.is_cuda and ssc_logit.dtype == torch.float32 and ssc_logit.dim() == 5):
            raise RuntimeError("OccDepth.class_map: expected CUDA fp32 logits [B, C, X, Y, Z]")
        x = ssc_logit.contiguous()
        B, Cn = x.shape[:2]
        S = x[0, 0].numel()
        out = torch.empty((B,) + tuple(x.shape[2:]), dtype=torch.uint16, device=x.device)
        lut = None
        if inv_map is not None:
            import numpy as np
            lut = np.ascontiguousarray(np.asarray(inv_map).astype(np.int32))
            if lut.shape != (Cn,):
                raise ValueError("OccDepth.class_map: inv_map must hold one label id per class")
        lut_p = None if lut is None else lut.ctypes.data
        if probabilities:
            probs = torch.empty(x.shape, dtype=torch.float16, device=x.device)
            _lib.check(_lib.lib().occd_class_probs(x.data_ptr(), out.data_ptr(), probs.data_ptr(), B, Cn, S, lut_p,
                                                   _lib.stream_ptr()), "occd_class_probs")
            return out, probs
        if confidence:
            conf = torch.empty(out.shape, dtype=torch.float16, device=x.device)
            _lib.check(_lib.lib().occd_argmax_classes_conf(x.data_ptr(), out.data_ptr(), conf.data_ptr(), B, Cn, S,
                                                           lut_p, _lib.stream_ptr()), "occd_argmax_classes_conf")
            return out, conf
        _lib.check(_lib.lib().occd_argmax_classes(x.data_ptr(), out.data_ptr(), B, Cn, S, lut_p, _lib.stream_ptr()),
                   "occd_argmax_classes")
        return out

    def predict(self, batch, inv_map=None):
        """forward + class map: returns (y_pred uint16 [B, X, Y, Z], the forward's output dict)"""
        res = self.forward(batch)
        return self.class_map(res["ssc_logit"], inv_map), res

    def step(self, *a, **k):
        raise NotImplementedError("occdepth_b200 implements the forward and the evaluation hooks only (training is "
                                  "out of scope)")

    # ---- evaluation: the metric side of the reference's test / validation steps (OccDepth.py:539-580) -----------
    def slab_x_range(self):
        """full-resolution X planes [lo, hi) of the class map predict_classes returned on this rank under
        enable_slab_parallel, from its plan; None without the partition"""
        if self.__dict__.get("slab_ctx") is None:
            return None
        (plan, *_), = self._class_plans().values()
        return plan.x_range

    def _count(self, metric, batch):
        """the class map of `batch` (training class ids: no remap) counted against batch["target"] on the device;
        under the slab partition, this rank's X-slab of both"""
        y = self.predict_classes(batch)
        target = batch["target"]
        xr = self.slab_x_range()
        if xr is not None:
            target = target[:, xr[0]:xr[1]]
        metric.add_batch(y, target.contiguous())

    def sem_decay_scale(self):
        """the sem-scal loss factor of OccDepth.step (OccDepth.py:467-470)"""
        if self.sem_step_decay_loss:
            return max(0.1, (1 - self.cur_batch / self.total_batch))
        return 1.0

    @staticmethod
    def eval_losses_enabled():
        """OCCDEPTH_EVAL_LOSSES=1: test_step / validation_step also compute and log the reference's losses (read
        when a step runs, so an unmodified evaluation script can switch it on)"""
        v = os.environ.get("OCCDEPTH_EVAL_LOSSES", "0")
        if v not in ("0", "1"):
            raise ValueError("OCCDEPTH_EVAL_LOSSES must be '0' or '1'")
        return v == "1"

    def _eval_step(self, batch, step_type, metric):
        if not self.eval_losses_enabled():
            self._count(metric, batch)
            return
        if self.__dict__.get("slab_ctx") is not None:
            raise NotImplementedError("OCCDEPTH_EVAL_LOSSES=1 under enable_slab_parallel: the losses of an X-slab "
                                      "partition are not computed (unset OCCDEPTH_EVAL_LOSSES to count the metrics)")
        # the reference's OccDepth.step: one forward, the losses in its order, the metrics, then the total
        out = self(batch)
        losses = step_losses(self, out, batch, step_type)
        total = losses.pop(step_type + "/loss")
        for key, value in losses.items():
            self.log(key, value, on_epoch=True, sync_dist=True)
        metric.add_batch(self.class_map(out["ssc_logit"]), batch["target"].contiguous())
        self.log(step_type + "/loss", total, on_epoch=True, sync_dist=True)

    def test_step(self, batch, batch_idx):
        self._eval_step(batch, "test", self.test_metrics)

    def validation_step(self, batch, batch_idx):
        self._eval_step(batch, "val", self.val_metrics)

    @staticmethod
    def _sum_over_ranks(*metrics):
        """under a process group of several ranks, every rank's counters become the sum over ranks (the reference
        reports each rank's own shard under DDP; here every rank reports the whole split)"""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            for m in metrics:
                m.all_reduce()

    def validation_epoch_end(self, outputs):
        metric_list = [("train", self.train_metrics), ("val", self.val_metrics)]
        self._sum_over_ranks(*(m for _, m in metric_list))
        for prefix, metric in metric_list:
            stats = metric.get_stats()
            for i, class_name in enumerate(self.class_names):
                self.log("{}_SemIoU/{}".format(prefix, class_name), stats["iou_ssc"][i], sync_dist=True)
            self.log("{}/mIoU".format(prefix), stats["iou_ssc_mean"], sync_dist=True)
            self.log("{}/IoU".format(prefix), stats["iou"], sync_dist=True)
            self.log("{}/Precision".format(prefix), stats["precision"], sync_dist=True)
            self.log("{}/Recall".format(prefix), stats["recall"], sync_dist=True)
            metric.reset()

    def test_epoch_end(self, outputs):
        classes = self.class_names
        metric_list = [("test", self.test_metrics)]
        self._sum_over_ranks(*(m for _, m in metric_list))
        for prefix, metric in metric_list:
            print("{}======".format(prefix))
            stats = metric.get_stats()
            print("Precision={:.4f}, Recall={:.4f}, IoU={:.4f}".format(
                stats["precision"] * 100, stats["recall"] * 100, stats["iou"] * 100))
            print("class IoU: {}, ".format(classes))
            print(" ".join(["{:.4f}, "] * len(classes)).format(*(stats["iou_ssc"] * 100).tolist()))
            print("mIoU={:.4f}".format(stats["iou_ssc_mean"] * 100))
            metric.reset()
