"""Generates tests/golden/* by running the UNMODIFIED reference (imported through oracle/ref_import.py) on seeded
inputs and weights:  OCCDEPTH_REFERENCE=<checkout of the original project> python -m oracle.gen_golden

Each fixture stores the inputs (or the seed that regenerates them), the seed of `synth.seed_weights_`, and the
reference outputs (fp16-safe small tensors kept as fp32).
"""
import copy
import os

import torch
import torch.nn as nn

from . import ref_import, synth

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def sfa_cases():
    return [("kitti", 2, 1, 16), ("NYU", 2, 1, 16), ("kitti", 1, 1, 8), ("kitti", 2, 5, 8), ("kitti", 3, 1, 8)]


def gen_sfa(ref):
    out = {}
    scene, ps, h, w = (12, 10, 8), 2, 9, 17
    N = 6 * 5 * 4
    for i, (ds, V, P, C) in enumerate(sfa_cases()):
        g = torch.Generator().manual_seed(100 + i)
        x2d = torch.randn(V, C, h, w, generator=g)
        pix, fov = synth.random_indices(N, w, h, n_views=V, P=P, seed=200 + i, margin=(4, 3))
        y = ref.SFA.SFA(scene, ds, ps)(x2d, pix.clone(), fov.clone()).contiguous()
        out["case%d" % i] = dict(dataset=ds, x2d=x2d, pix=pix, fov=fov, out=y, scene=scene, ps=ps)
    torch.save(out, os.path.join(OUT, "sfa.pt"))


def gen_unet3d(ref):
    with ref_import.quiet():
        mk = ref.unet3d_kitti.UNet3D(5, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=True, cascade_cls=True,
                                     occluded_cls=True).eval()
        mn = ref.unet3d_nyu.UNet3D(5, nn.BatchNorm3d, 16, (12, 8, 12), context_prior=True, cascade_cls=False).eval()
    synth.seed_weights_(mk, 11)
    synth.seed_weights_(mn, 12)
    g = torch.Generator().manual_seed(3)
    xk = torch.randn(1, 16, 16, 16, 8, generator=g)
    xn = torch.randn(1, 16, 12, 8, 12, generator=g)
    with torch.no_grad():
        ok, on = mk({"x3d": xk}), mn({"x3d": xn})
    keep = ("ssc_logit", "occ_logit", "occluded_logit", "P_logits")
    torch.save(dict(kitti=dict(x=xk, seed=11, out={k: v for k, v in ok.items() if k in keep}),
                    nyu=dict(x=xn, seed=12, out={k: v for k, v in on.items() if k in keep})),
               os.path.join(OUT, "unet3d.pt"))


def gen_occdepth(ref):
    full = (32, 32, 16)
    cfg = synth.occdepth_cfg(full_scene_size=full, feature=16, feature_2d_oc=16, n_classes=6,
                             backbone_2d_name="tf_efficientnet_b3_ns")
    with ref_import.quiet():
        m = ref.OccDepth.OccDepth(["c"] * 6, torch.ones(6), full_scene_size=full, project_res=["1", "2", "4", "8"],
                                  config=cfg).eval()
    synth.seed_weights_(m, 21)
    H, W = 33, 49
    g = torch.Generator().manual_seed(0)
    img = torch.randn(1, 2, 3, H, W, generator=g)
    pix, fov = synth.random_indices(16 * 16 * 8, W, H, n_views=2, P=1, seed=5, margin=(10, 6))
    with torch.no_grad():
        out = m({"img": img, "projected_pix_2": [pix], "fov_mask_2": [fov]})
        feats = m.net_rgb(img[:, 0])
    torch.save(dict(img=img, pix=pix, fov=fov, seed=21, cfg=dict(cfg), ssc_logit=out["ssc_logit"],
                    occ_logit=out["occ_logit"], feat_1_8=feats["1_8"], feat_1_1_mean=feats["1_1"].mean((2, 3))),
               os.path.join(OUT, "occdepth_small.pt"))


def vox2pix_cases():
    """(name, cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id): a KITTI-like rig with a
    slightly rotated pose (so every term of the pose matrix matters), an NYU-like one, and a camera INSIDE the volume
    (voxels behind it and one column of centres in the camera plane: z <= 0, division by zero)"""
    import math
    import numpy as np

    def rot(ax, a):
        c, s = math.cos(a), math.sin(a)
        R = np.eye(3)
        i, j = [(1, 2), (0, 2), (0, 1)][ax]
        R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
        return R
    base = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0.0]])
    E1 = np.eye(4)
    E1[:3, :3] = rot(0, 0.03) @ rot(1, -0.02) @ rot(2, 0.01) @ base
    E1[:3, 3] = [0.011, -0.083, -0.271]
    K1 = np.array([[707.0912, 0, 601.8873], [0, 707.0912, 183.1104], [0, 0, 1.0]])
    E2 = np.eye(4)
    E2[:3, :3] = rot(0, -0.4) @ rot(2, 0.7)
    E2[:3, 3] = [0.3, -0.2, 1.1]
    K2 = np.array([[518.8579, 0, 320.0], [0, 518.8579, 240.0], [0, 0, 1.0]])
    E3 = np.eye(4)
    E3[:3, :3] = base
    E3[:3, 3] = [0.0, 0.0, -0.75]         # cam z = lidar x - 0.75: the centres at x = 0.75 lie exactly in the camera plane
    return [("kitti_p0", E1, K1, np.array([0, -6.4, -2.0]), 0.4, 1220, 370, (12.8, 12.8, 3.2), 0),
            ("kitti_p3", E1, K1, np.array([0, -6.4, -2.0]), 0.8, 1220, 370, (12.8, 12.8, 3.2), 3),
            ("nyu_p8", E2.astype(np.float32), K2, np.array([-1.2, -1.0, 0.1]), 0.16, 640, 480, (2.4, 2.4, 1.44), 8),
            ("plane_p1", E3, K1, np.array([0.0, -2.0, -1.0]), 0.5, 1220, 370, (4.0, 4.0, 2.0), 1)]


def gen_vox2pix():
    helpers = ref_import.data_helpers()
    out = {}
    for name, E, K, org, vs, W, H, scene, pid in vox2pix_cases():
        pix, fov, z = helpers.vox2pix(E, K, org, vs, W, H, scene, pid)
        out[name] = dict(cam_E=torch.from_numpy(E.copy()), cam_k=torch.from_numpy(K.copy()),
                         vox_origin=torch.from_numpy(org.copy()), voxel_size=vs, img_W=W, img_H=H,
                         # pixel indices stored as int32 where they fit (the projection returns int64; the tests
                         # compare values), which keeps the file under 1 MB
                         scene_size=scene, pattern_id=pid, fov=torch.from_numpy(fov),
                         pix=torch.from_numpy(pix).to(torch.int32) if abs(pix).max() < 2 ** 31 - 1 else torch.from_numpy(pix),
                         pix_z=torch.from_numpy(z))
    torch.save(out, os.path.join(OUT, "vox2pix.pt"))


def state_dict_cases():
    """(name, builder(namespace of occdepth.models modules) -> module): the modules whose state_dict layout released
    checkpoints depend on; the same builders run on the reference's modules and on occdepth_b200.models"""
    def occdepth(variant):
        def build(ns):
            if variant == "nyu_flosp":
                cfg = synth.occdepth_cfg(dataset="NYU", full_scene_size=(60, 36, 60), project_scale=1, feature=200,
                                         feature_2d_oc=200, n_classes=12, cascade_cls=False)
            else:
                cfg = synth.occdepth_cfg(trans_2d_to_3d="flosp_depth" if variant.endswith("depth") else "flosp")
            kw = dict(full_scene_size=cfg.full_scene_size, project_res=["1", "2", "4", "8"], config=cfg)
            return ns.OccDepth.OccDepth(["c"] * cfg.n_classes, torch.ones(cfg.n_classes), **kw)
        return build

    def flosp(ds):
        def build(ns):
            c = copy.deepcopy(ns.flosp_conf[ds])
            c.update(scene_size=(256, 256, 32) if ds == "kitti" else (60, 36, 60),
                     project_scale=2 if ds == "kitti" else 1, return_depth=False)
            return ns.flosp_depth.FlospDepth(**c)
        return build
    kw3 = dict(context_prior=True, cascade_cls=True, occluded_cls=True)
    cases = [
        ("unet3d_kitti", lambda ns: ns.unet3d_kitti.UNet3D(20, nn.BatchNorm3d, (256, 256, 32), 64, 2, **kw3)),
        ("unet3d_nyu", lambda ns: ns.unet3d_nyu.UNet3D(12, nn.BatchNorm3d, 200, (60, 36, 60))),
        ("unet3d_kitti_ps1", lambda ns: ns.unet3d_kitti.UNet3D(20, nn.BatchNorm3d, (128, 128, 16), 32, 1)),
    ]
    for bb in ("tf_efficientnet_b3_ns", "tf_efficientnet_b4_ns", "tf_efficientnet_b5_ns", "tf_efficientnet_b7_ns"):
        cases.append(("unet2d_" + bb, lambda ns, bb=bb: ns.unet2d.UNet2D.build(
            out_feature=64, use_decoder=True, backbone_2d_name=bb, return_up_feats=1)))
    cases += [("flosp_depth_kitti", flosp("kitti")), ("flosp_depth_NYU", flosp("NYU"))]
    cases += [("occdepth_" + v, occdepth(v)) for v in ("kitti_flosp", "kitti_flosp_depth", "nyu_flosp")]
    return cases


def state_dict_layout(m):
    """(number of entries, digest of the ordered keys, shapes and dtypes) of a module's state_dict"""
    import hashlib
    sd = m.state_dict()
    text = "\n".join("%s %s %s" % (k, tuple(v.shape), v.dtype) for k, v in sd.items())
    return [len(sd), hashlib.sha256(text.encode()).hexdigest()]


def gen_state_dicts(ref):
    """state_dict layout (state_dict_layout) of the reference's modules and its flosp_depth_conf_map ->
    state_dict_layout.json (what tests/test_state_dict_compat.py compares occdepth_b200.models against)"""
    import json
    import occdepth.models.flosp_depth as rfd
    ref.flosp_conf = rfd.flosp_depth_conf_map
    out = {"conf_map": copy.deepcopy(rfd.flosp_depth_conf_map), "modules": {}}
    saved = copy.deepcopy(rfd.flosp_depth_conf_map)
    for name, build in state_dict_cases():
        with ref_import.quiet():
            m = build(ref)
        for k in rfd.flosp_depth_conf_map:       # the reference mutates its conf dicts in place
            rfd.flosp_depth_conf_map[k].clear()
            rfd.flosp_depth_conf_map[k].update(copy.deepcopy(saved[k]))
        out["modules"][name] = state_dict_layout(m)
    with open(os.path.join(OUT, "state_dict_layout.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


PIN_SAMPLE = 1 << 10


def pin_index(numel, seed=0):
    """the fixed seeded sample of flat indices pin_sample keeps of a tensor with `numel` elements"""
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:PIN_SAMPLE].sort().values


def pin_sample(t):
    """a large tensor -> its shape and the values at pin_index; small tensors whole"""
    t = t.detach().contiguous()
    if t.numel() <= PIN_SAMPLE:
        return t
    return {"shape": tuple(t.shape), "values": t.reshape(-1)[pin_index(t.numel())].clone()}


def pin_digest(a):
    import hashlib
    import numpy as np
    a = np.ascontiguousarray(a)
    return "%s|%s|%s" % (a.dtype.str, "x".join(map(str, a.shape)), hashlib.sha256(a.tobytes()).hexdigest())


# inputs of the pinned cases, regenerated from seeds by the generator and by tests/test_oracle_vs_reference.py
SFA_CASES = [("kitti", 2, 1), ("kitti", 1, 1), ("NYU", 2, 1), ("kitti", 2, 5), ("kitti", 3, 1)]
FLOSP_HW = (96, 320)


def sfa_pin_inputs(V, P):
    x2d = torch.randn(V, 16, 11, 23, generator=torch.Generator().manual_seed(0))
    pix, fov = synth.random_indices(8 * 6 * 4, 23, 11, n_views=V, P=P, seed=3, margin=(5, 4))
    return x2d, pix, fov


def blocks_pin_input():
    return torch.randn(1, 16, 8, 10, 6, generator=torch.Generator().manual_seed(0))


def unet3d_pin_inputs():
    g = torch.Generator().manual_seed(1)
    return torch.randn(1, 16, 16, 16, 8, generator=g), torch.randn(1, 16, 12, 8, 12, generator=g)


def unet2d_pin_input():
    return torch.randn(1, 3, 38, 45, generator=torch.Generator().manual_seed(2))


def occdepth_small_pin_inputs():
    full = (32, 32, 16)
    cfg = synth.occdepth_cfg(full_scene_size=full, feature=16, feature_2d_oc=16, n_classes=6,
                             backbone_2d_name="tf_efficientnet_b3_ns")
    img = torch.randn(1, 2, 3, 33, 49, generator=torch.Generator().manual_seed(0))
    pix, fov = synth.random_indices(16 * 16 * 8, 49, 33, n_views=2, P=1, seed=5, margin=(10, 6))
    return full, cfg, {"img": img, "projected_pix_2": [pix], "fov_mask_2": [fov]}


def flosp_pin_inputs(conf_map):
    conf = copy.deepcopy(conf_map["kitti"])
    H, W = FLOSP_HW
    conf.update(scene_size=(64, 64, 8), project_scale=2, return_depth=True, final_dim=(H, W), output_channels=16,
                x_bound=[0, 12.8, 0.2], y_bound=[-6.4, 6.4, 0.2], z_bound=[-2, -0.4, 0.2], d_bound=[2.0, 18.0, 0.5],
                depth_net_conf=dict(in_channels=16, mid_channels=32))
    K, Ts = synth.kitti_calib(W, H, focal=220.0)
    feat = torch.randn(1, 2, 16, H // 8, W // 8, generator=torch.Generator().manual_seed(4))
    cam_k = [torch.from_numpy(K).unsqueeze(0).repeat(2, 1, 1)]
    T = [torch.stack([torch.from_numpy(t) for t in Ts])]
    ida = [torch.eye(4).unsqueeze(0).repeat(2, 1, 1)]
    return conf, feat, cam_k, T, ida


def nyu_virtual_pin_inputs():
    full = (12, 8, 12)
    cfg = synth.occdepth_cfg(dataset="NYU", full_scene_size=full, project_scale=1, feature=16, feature_2d_oc=16,
                             n_classes=6, cascade_cls=False, backbone_2d_name="tf_efficientnet_b3_ns")
    H, W = 32, 64
    g = torch.Generator().manual_seed(0)
    img = torch.randn(1, 1, 3, H, W, generator=g)
    depth = torch.rand(1, 1, H, W, generator=g) * 7.5 + 0.5
    depth[0, 0, 3, 5] = 0.0          # exercises the inf -> 0 disparity rule (OccDepth.py:248)
    pix, fov = synth.random_indices(full[0] * full[1] * full[2], W, H, n_views=2, P=1, seed=1, margin=(8, 6))
    return full, cfg, {"img": img, "gt_depth": depth, "virtual_bf": [torch.tensor(51.88579 * W / 640.0)],
                       "vox_origin": torch.zeros(1, 3, dtype=torch.float64), "projected_pix_1": [pix],
                       "fov_mask_1": [fov]}


def block_modules(ns):
    """the three small 3-D building blocks of tests/test_oracle_vs_reference.py, from a namespace with `modules`"""
    return (ns.modules.Process(16, nn.BatchNorm3d, 0.1, dilations=[1, 2, 3]).eval(),
            ns.modules.Downsample(16, nn.BatchNorm3d, 0.1).eval(), ns.modules.Upsample(32, 16, nn.BatchNorm3d, 0.1).eval())


def gen_reference_pins(ref):
    """reference outputs behind tests/test_oracle_vs_reference.py -> reference_pins.pt.  Inputs are regenerated
    from seeds (the *_pin_input(s) functions above), weights are synth.seed_weights_ fills (reproducible on
    occdepth_b200.models, which has the same state_dict keys); large outputs are kept as a fixed seeded sample
    (pin_sample), the projection's outputs as digests of their bytes."""
    import occdepth.models.flosp_depth as rfd
    out = {}
    with ref_import.quiet(), torch.no_grad():
        for ds, V, P in SFA_CASES:
            x2d, pix, fov = sfa_pin_inputs(V, P)
            out["sfa_%s_%d_%d" % (ds, V, P)] = ref.SFA.SFA((16, 12, 8), ds, 2)(x2d, pix.clone(), fov.clone()).contiguous()
        x = blocks_pin_input()
        proc, down, up = block_modules(ref)
        for i, m in enumerate((proc, down, up)):
            synth.seed_weights_(m, 40 + i)
        y = down(x)
        out["blocks"] = {"process": proc(x), "downsample": y, "upsample": up(y)}
        xk, xn = unet3d_pin_inputs()
        mk = ref.unet3d_kitti.UNet3D(5, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=True, cascade_cls=True,
                                     occluded_cls=True).eval()
        mn = ref.unet3d_nyu.UNet3D(5, nn.BatchNorm3d, 16, (12, 8, 12), context_prior=True, cascade_cls=False).eval()
        synth.seed_weights_(mk, 31)
        synth.seed_weights_(mn, 32)
        out["unet3d_kitti"] = {k: pin_sample(v) for k, v in mk({"x3d": xk}).items()}
        out["unet3d_nyu"] = {k: pin_sample(v) for k, v in mn({"x3d": xn}).items()}
        m = ref.unet2d.UNet2D.build(out_feature=16, use_decoder=True, backbone_2d_name="tf_efficientnet_b3_ns",
                                    return_up_feats=1).eval()
        synth.seed_weights_(m, 33)
        out["unet2d"] = {k: pin_sample(v) for k, v in m(unet2d_pin_input()).items()}
        full, cfg, batch = occdepth_small_pin_inputs()
        m = ref.OccDepth.OccDepth(class_names=["c"] * 6, class_weights=torch.ones(6), full_scene_size=full,
                                  project_res=["1", "2", "4", "8"], config=cfg).eval()
        synth.seed_weights_(m, 34)
        out["occdepth_small"] = {k: pin_sample(v) for k, v in m(batch).items()}
        conf, feat, cam_k, T, ida = flosp_pin_inputs(rfd.flosp_depth_conf_map)
        m = synth.seed_weights_(ref.flosp_depth.FlospDepth(**conf).eval(), 5)
        want, want_d = m(feat, cam_k, T, ida, None)
        out["flosp_depth"] = {"cover": float((want > 0).float().mean()), "out": pin_sample(want),
                              "depth": pin_sample(want_d)}
        full, cfg, batch = nyu_virtual_pin_inputs()
        m = ref.OccDepth.OccDepth(["c"] * 6, torch.ones(6), full_scene_size=full, project_res=["1", "2", "4", "8"],
                                  config=cfg).eval()
        synth.seed_weights_(m, 3)
        out["occdepth_nyu_virtual_view"] = {k: pin_sample(v) for k, v in m(batch).items()}
    helpers = ref_import.data_helpers()
    dig = {}
    for pid in (0, 1, 3, 6, 8):
        for name, E, K, org, vs, W, H, scene, _ in vox2pix_cases():
            dig["%s_%d" % (name, pid)] = [pin_digest(a) for a in helpers.vox2pix(E, K, org, vs, W, H, scene, pid)]
    out["vox2pix_digests"] = dig
    torch.save(out, os.path.join(OUT, "reference_pins.pt"))

def main():
    os.makedirs(OUT, exist_ok=True)
    ref = ref_import.modules()
    torch.manual_seed(0)
    gen_sfa(ref)
    gen_unet3d(ref)
    gen_occdepth(ref)
    gen_vox2pix()
    gen_state_dicts(ref)
    gen_reference_pins(ref)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
