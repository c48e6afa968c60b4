"""Drop-in for the reference `occdepth/models/flosp_depth/flosp_depth.py`: Mlp :159, SELayer :186, DepthNet :201-257,
FlospDepth :324-608 (+ the conf dicts of flosp_depth_conf_{kitti,nyu}.py).

DepthNet's convolutions run on the wgmma implicit-GEMM kernel; the frustum grid (f2v/frustum_grid_generator.py) is
never materialised -- `occd_frustum_sample_fwd` computes each voxel's sampling coordinate on the fly and fuses the
trilinear sampling of the depth distribution, of the all-ones mask volume and the per-camera masked mean.
"""
import torch
import torch.nn as nn

from ... import _lib
from ...engine import FnOp, fold_bn
from .._base import B200Module

flosp_depth_conf_kitti = {
    "x_bound": [0, 51.2, 0.2], "y_bound": [-25.6, 25.6, 0.2], "z_bound": [-2, 4.4, 0.2], "d_bound": [2.0, 54.0, 0.5],
    "final_dim": (370, 1220), "output_channels": 64, "downsample_factor": 8,
    "depth_net_conf": dict(in_channels=64, mid_channels=128), "disc_cfg": dict(mode="LID"), "agg_voxel_mode": "mean",
}
flosp_depth_conf_nyu = {
    "x_bound": [0, 4.8, 0.08], "y_bound": [-2.4, 2.4, 0.08], "z_bound": [0, 2.88, 0.08], "d_bound": [0, 10, 0.08],
    "final_dim": (480, 640), "output_channels": 64, "downsample_factor": 8,
    "depth_net_conf": dict(in_channels=64, mid_channels=128), "disc_cfg": dict(mode="LID"), "agg_voxel_mode": "mean",
}
flosp_depth_conf_map = {"NYU": flosp_depth_conf_nyu, "kitti": flosp_depth_conf_kitti}


class BasicBlock(nn.Module):
    """parameter layout of mmdet 2.20 BasicBlock (flosp_depth.py:4,219-221): conv1, bn1, conv2, bn2"""

    def __init__(self, inplanes, planes):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.ReLU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.drop1 = nn.Dropout(drop)
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop2 = nn.Dropout(drop)


class SELayer(nn.Module):
    def __init__(self, channels, act_layer=nn.ReLU, gate_layer=nn.Sigmoid):
        super().__init__()
        self.conv_reduce = nn.Conv2d(channels, channels, 1, bias=True)
        self.act1 = act_layer()
        self.conv_expand = nn.Conv2d(channels, channels, 1, bias=True)
        self.gate = gate_layer()


class DepthNet(nn.Module):
    def __init__(self, in_channels, mid_channels, context_channels, depth_channels, infer_mode=False):
        super(DepthNet, self).__init__()
        self.reduce_conv = nn.Sequential(
            nn.Conv2d(in_channels, mid_channels, kernel_size=3, stride=1, padding=1),
            nn.BatchNorm2d(mid_channels),
            nn.ReLU(inplace=True))
        self.mlp = Mlp(1, mid_channels, mid_channels)
        self.se = SELayer(mid_channels)
        self.depth_conv = nn.Sequential(BasicBlock(mid_channels, mid_channels), BasicBlock(mid_channels, mid_channels),
                                        BasicBlock(mid_channels, mid_channels))
        self.depth_pred = nn.Conv2d(mid_channels, depth_channels, kernel_size=1, stride=1, padding=0)
        self.infer_mode = infer_mode


class FlospDepth(B200Module):
    def __init__(self, x_bound, y_bound, z_bound, d_bound, final_dim, downsample_factor, output_channels,
                 depth_net_conf, scene_size, project_scale, return_depth, agg_voxel_mode="mean", infer_mode=False,
                 **kwargs):
        super().__init__()
        self.downsample_factor = downsample_factor
        self.d_bound = d_bound
        self.final_dim = final_dim
        self.output_channels = output_channels
        self.depth_channels = int((self.d_bound[1] - self.d_bound[0]) / self.d_bound[2])
        self.scene_size = scene_size
        self.project_scale = project_scale
        self.infer_mode = infer_mode
        self.depth_net_conf = depth_net_conf
        self.depth_net = nn.Sequential(DepthNet(depth_net_conf["in_channels"], depth_net_conf["mid_channels"],
                                                self.output_channels, self.depth_channels, infer_mode=infer_mode))
        self.bounds = [x_bound, y_bound, z_bound]
        self.register_buffer("voxel_size", torch.Tensor([row[2] * project_scale for row in self.bounds]))
        self.register_buffer("voxel_coord",
                             torch.Tensor([row[0] + row[2] / 2.0 * project_scale for row in self.bounds]))
        self.register_buffer("voxel_num",
                             torch.LongTensor([(row[1] - row[0]) / row[2] / project_scale for row in self.bounds]))
        self.return_depth = return_depth
        self.agg_voxel_mode = agg_voxel_mode
        if agg_voxel_mode not in ("mean", "sum"):
            raise NotImplementedError("agg_voxel_mode: {}".format(agg_voxel_mode))

    # ---- host-side camera preprocessing (what FlospDepth.forward / FrustumGridGenerator do with torch on the
    # ---- host for 4x4 matrices, flosp_depth.py:466-541, frustum_grid_generator.py:20-67) ----
    def _grid_to_lidar(self, vox_origin):
        vn = [int(v) for v in self.voxel_num.tolist()]
        if vox_origin is not None:    # NYU: bounds rebuilt from batch item 0's origin every forward (:466-518)
            o = [float(vox_origin[0][k]) for k in range(3)]
            ext = (4.8, 4.8, 2.88)
            bounds = [[o[k], o[k] + ext[k], 0.08] for k in range(3)]
            vn = [int((b[1] - b[0]) / b[2] / self.project_scale) for b in bounds]
        else:
            bounds = self.bounds
        pc_min = torch.tensor([b[0] for b in bounds], dtype=torch.float32)
        pc_max = torch.tensor([b[1] for b in bounds], dtype=torch.float32)
        vs = (pc_max - pc_min) / torch.tensor(vn, dtype=torch.float32)
        G = torch.eye(4, dtype=torch.float32)
        G[0, 0], G[1, 1], G[2, 2] = vs[0], vs[1], vs[2]
        G[:3, 3] = pc_min
        return G, vn

    def camera_tables(self, cam_k, T_velo_2_cam, ida_mats, vox_origin, n_cams):
        """-> (cams [B, V, 40] fp32, scaled_pixel_size [B*V, 1] fp32, (X, Y, Z))"""
        G, vn = self._grid_to_lidar(vox_origin)
        B = len(cam_k)
        cams = torch.zeros(B, n_cams, 40, dtype=torch.float32)
        sps = torch.zeros(B * n_cams, 1, dtype=torch.float32)
        for b in range(B):
            K = cam_k[b].to(torch.float32).cpu()
            T = T_velo_2_cam[b].to(torch.float32).cpu()
            A = ida_mats[b].to(torch.float32).cpu()
            for v in range(n_cams):
                K4 = torch.zeros(4, 4)
                K4[:3, :3] = K[v]
                K4[3, 3] = 1
                inv = torch.inverse(K4)
                sps[b * n_cams + v, 0] = torch.norm(torch.stack([inv[0, 0], inv[1, 1]])) * 1000.0
                cams[b, v, :12] = (T[v] @ G)[:3].reshape(-1)
                cams[b, v, 12:24] = K4[:3].reshape(-1)
                cams[b, v, 24:] = A[v].reshape(-1)
        return cams, sps, vn

    def emit(self, plan, x_rgb, batch, B, V, n_cams=None, window=None):
        """x_rgb: {"1_s": CL [B*V,1,h,w,C]} -> prior fp32 [B, X*Y*Z] (voxel order of the lift output).
        window (x0, Xl): only the planes [x0, x0 + Xl) of the X axis, as [B, Xl*Y*Z] (the X-slab partition: DepthNet
        runs whole on every rank, the frustum sampling on this rank's slab).  The plan's input buffers are kept in
        self.plan_state() until the next emit."""
        L = _lib.lib()
        dev = plan.device
        n_cams = V if n_cams is None else n_cams
        feat = x_rgb["1_%d" % self.downsample_factor]
        BV, _, h, w = feat.dims
        assert BV == B * V
        dn = self.depth_net[0]
        mid = dn.depth_pred.in_channels
        Dn = self.depth_channels
        wr, br = fold_bn(dn.reduce_conv[0].weight, dn.reduce_conv[0].bias, dn.reduce_conv[1])
        x = plan.conv(feat, wr.unsqueeze(2), br, padding=(0, 1, 1), act="relu", name="depthnet.reduce")
        sps = torch.zeros(BV, 1, dtype=torch.float32, device=dev)

        def fc(inp, lin_w, lin_b, n_in, n_out, act, nm):
            wt = lin_w.detach().float().reshape(n_out, n_in).contiguous()
            bt = lin_b.detach().float().contiguous()
            o = torch.empty(BV, n_out, dtype=torch.float32, device=dev)
            plan.add(FnOp(lambda st: L.occd_fc_fwd(inp.data_ptr(), wt.data_ptr(), bt.data_ptr(), o.data_ptr(), BV, n_in,
                                                   n_out, act, st), nm, keep=(inp, wt, bt, o)))
            return o

        h1 = fc(sps, dn.mlp.fc1.weight, dn.mlp.fc1.bias, 1, mid, _lib.ACT_RELU, "depthnet.mlp.fc1")
        h2 = fc(h1, dn.mlp.fc2.weight, dn.mlp.fc2.bias, mid, mid, _lib.ACT_NONE, "depthnet.mlp.fc2")
        g1 = fc(h2, dn.se.conv_reduce.weight, dn.se.conv_reduce.bias, mid, mid, _lib.ACT_RELU, "depthnet.se.reduce")
        gate = fc(g1, dn.se.conv_expand.weight, dn.se.conv_expand.bias, mid, mid, _lib.ACT_SIGMOID, "depthnet.se.gate")
        plan.add(FnOp(lambda st, xg=x: L.occd_channel_scale(xg.ptr, gate.data_ptr(), plan.lib_dtype, BV, h * w, mid,
                                                            xg.cstride, st),
                      "depthnet.se.scale", keep=(x, gate)))      # xg bound now: `x` is rebound by the blocks below
        for i, blk in enumerate(dn.depth_conv):
            w1, b1 = fold_bn(blk.conv1.weight, None, blk.bn1)
            y = plan.conv(x, w1.unsqueeze(2), b1, padding=(0, 1, 1), act="relu", name="depthnet.block%d.conv1" % i)
            w2, b2 = fold_bn(blk.conv2.weight, None, blk.bn2)
            x = plan.conv(y, w2.unsqueeze(2), b2, padding=(0, 1, 1), act="relu", res1=x,
                          name="depthnet.block%d.conv2" % i)
        logits = torch.empty(BV, Dn, 1, h, w, dtype=torch.float32, device=dev)
        wp = dn.depth_pred.weight.detach().float()
        plan.conv(x, wp.unsqueeze(2), dn.depth_pred.bias.detach().float(), out1=logits, out1_mode="planar",
                  no_out0=True, name="depthnet.depth_pred")
        prob = torch.empty(BV, Dn, h, w, dtype=torch.float32, device=dev)
        plan.add(FnOp(lambda st: L.occd_softmax_planar(logits.data_ptr(), prob.data_ptr(), BV, Dn, h * w, st),
                      "depth.softmax", keep=(logits, prob)))
        vox_origin = batch.get("vox_origin") if isinstance(batch, dict) else None
        _, vn = self._grid_to_lidar(vox_origin if vox_origin is not None else None)
        X, Y, Z = vn
        x0, Xl = window if window is not None else (0, X)
        if not (Xl > 0 and 0 <= x0 <= X - Xl):
            raise ValueError("FlospDepth: window [%d, %d) is outside the %d X planes of the grid" % (x0, x0 + Xl, X))
        cams = torch.zeros(B, n_cams, 40, dtype=torch.float32, device=dev)
        # vn is baked into the plan's buffers; stage_inputs checks every batch against it
        state = {"sps": sps, "vn": tuple(vn), "cams": cams, "n_cams": n_cams, "window": (x0, Xl),
                 "prob": prob.view(B, V, Dn, h, w)}
        self.__dict__["_state"] = state
        prior = torch.empty(B, Xl * Y * Z, dtype=torch.float32, device=dev)
        perm = 1 if vox_origin is not None else 0      # NYU: x3ds_depth.permute(0,1,2,4,3), OccDepth.py:335-337
        H_img, W_img = self.final_dim
        mean_mode = 1 if self.agg_voxel_mode == "mean" else 0
        if self.infer_mode:
            # the caller supplies batch["grids"] (one (B, X, Y, Z, 3) grid per camera) and batch["scaled_pixel_size"]
            # (flosp_depth.py:564-565, OccDepth.py:310-317): staged into these static buffers before every replay
            # (only the window's rows are staged and read)
            grids = torch.zeros(B, n_cams, X * Y * Z, 3, dtype=torch.float32, device=dev)
            state["grids"] = grids
            for b in range(B):
                pb = prob[b * V:b * V + n_cams]
                plan.add(FnOp(lambda st, pb=pb, gb=grids[b], ob=prior[b]: L.occd_grid_sample_prior_window_fwd(
                    pb.data_ptr(), gb.data_ptr(), n_cams, Dn, h, w, X, Y, Z, x0, Xl, mean_mode, ob.data_ptr(), perm,
                    st), "grid_sample_prior", keep=(prob, grids, prior)))
        for b in range(B if not self.infer_mode else 0):
            pb = prob[b * V:b * V + n_cams]
            plan.add(FnOp(lambda st, pb=pb, cb=cams[b], ob=prior[b]: L.occd_frustum_sample_window_fwd(
                pb.data_ptr(), cb.data_ptr(), n_cams, Dn, h, w, X, Y, Z, x0, Xl, float(W_img), float(H_img),
                float(self.d_bound[0]), float(self.d_bound[1]), mean_mode,
                ob.data_ptr(), perm, st), "frustum_sample", keep=(prob, cams, prior)))
        return prior

    def plan_state(self):
        """input buffers and depth distribution of the plan the last emit() built"""
        return self.__dict__["_state"]

    def stage_inputs(self, batch, dev, state=None, item=None):
        """copy this batch's camera tables (or infer_mode grids) into the buffers of `state` (default: the plan the
        last emit() built); item: a one-frame batch's tables go to that batch item of the plan"""
        state = self.plan_state() if state is None else state
        if self.infer_mode:
            g = state["grids"]
            B, n_cams = g.shape[:2]
            x0, Xl = state["window"]
            grids = batch["grids"]
            for v in range(n_cams):
                gv = grids[v].to(torch.float32).reshape(B, -1, 3)
                plane = gv.shape[1] // state["vn"][0]
                g[:, v, x0 * plane:(x0 + Xl) * plane].copy_(gv[:, x0 * plane:(x0 + Xl) * plane], non_blocking=True)
            state["sps"].copy_(batch["scaled_pixel_size"].to(torch.float32).reshape(-1, 1), non_blocking=True)
            return
        cams, sps, vn = self.camera_tables(batch["cam_k"], batch["T_velo_2_cam"], batch["ida_mats"],
                                           batch.get("vox_origin"), state["n_cams"])
        if tuple(vn) != state["vn"]:
            # NYU: the voxel counts are re-derived from batch item 0's vox_origin every forward (flosp_depth.py:466-518)
            raise RuntimeError("FlospDepth: this batch's vox_origin gives a %r voxel grid, the plan was built for %r; "
                               "call invalidate_plans()" % (tuple(vn), state["vn"]))
        if item is None:
            state["cams"].copy_(cams, non_blocking=True)
            state["sps"].copy_(sps, non_blocking=True)
        else:
            n = state["n_cams"]
            state["cams"][item:item + 1].copy_(cams, non_blocking=True)
            state["sps"][item * n:(item + 1) * n].copy_(sps, non_blocking=True)

    def depth_prob(self, state=None):
        return (self.plan_state() if state is None else state)["prob"]

    def forward(self, img_feat, cam_k=None, T_velo_2_cam=None, ida_mats=None, vox_origin=None, grids=None,
                scaled_pixel_size=None):
        """stand-alone use: img_feat [B, n_cams, C, h, w] fp32 (CUDA) -> (B, 1, X, Y, Z) [, depth (B, n_cams, D, h, w)]"""
        from ...engine import CL, Plan, require_cuda
        require_cuda(img_feat, "FlospDepth.forward")
        if self.training:
            raise RuntimeError("FlospDepth: forward/inference only; call .eval()")
        B, V, C_, h, w = img_feat.shape
        key = (tuple(img_feat.shape), str(img_feat.device), vox_origin is not None, self.precision, self.param_stamp())
        ent = self._plans().get(key)
        batch = {"cam_k": cam_k, "T_velo_2_cam": T_velo_2_cam, "ida_mats": ida_mats}
        if self.infer_mode:
            batch = {"grids": grids, "scaled_pixel_size": scaled_pixel_size}
        if vox_origin is not None:
            batch["vox_origin"] = vox_origin
        if ent is None:
            self._plans().clear()
            plan = Plan(img_feat.device, precision=self.precision)
            xin = plan.alloc(B * V, 1, h, w, C_)
            with torch.no_grad():
                prior = self.emit(plan, {"1_%d" % self.downsample_factor: xin}, batch, B, V)
            plan.flosp_state = self.plan_state()
            ent = (plan, xin, prior)
            self._plans()[key] = ent
        plan, xin, prior = ent
        CL.from_planar(img_feat.reshape(B * V, C_, h, w), out=xin)
        self.stage_inputs(batch, img_feat.device, plan.flosp_state)
        plan.run()
        _, vn = self._grid_to_lidar(vox_origin)
        X, Y, Z = vn
        out = prior.clone().view(B, 1, X, Z, Y).permute(0, 1, 2, 4, 3) if vox_origin is not None \
            else prior.clone().view(B, 1, X, Y, Z)
        if self.return_depth:
            return out, self.depth_prob(plan.flosp_state).clone()
        return out
