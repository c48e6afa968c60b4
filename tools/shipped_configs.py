#!/usr/bin/env python
"""Forward time of every model configuration the original project ships (its config/*.yaml), at the shapes it was
trained on, in both arithmetic modes.

  python tools/shipped_configs.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [names...]

Prints one JSON line per (configuration, precision): ms per frame (CUDA events around K forwards, after W warm-up
forwards; that window is timed R times, the median is `ms_per_frame`, every window is listed), the card's name and
power limit read in the same run.  The image, projection indices, FOV masks and depth map are resident on the device
(`to_cuda`); the camera matrices stay in host memory, where the forward turns them into its per-camera tables.
Weights are module-default init with randomised BatchNorm statistics, inputs are seeded: the time does not depend on
the values.

`make_case` builds the model and a batch for one configuration; tests/test_gpu_shipped_configs.py uses it to compare
the forward with the CPU oracle at the same shapes.
"""
import argparse
import contextlib
import copy
import io
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KITTI_IMG = (376, 1370)            # H, W
KITTI_FULL = (256, 256, 32)
NYU_IMG = (480, 640)
NYU_FULL = (60, 36, 60)
PROJECT_RES = ["1", "2", "4", "8"]

# the fields of the shipped YAML files that change the forward
CONFIGS = {
    "nyu_b4_f100_2080ti": dict(   # NYU/multicam_flosp_crp_stereodepth_cascadecls_2080ti.yaml (released NYUv2 model)
        dataset="NYU", backbone_2d_name="tf_efficientnet_b4_ns", feature=100, trans_2d_to_3d="flosp", views=1,
        context_prior=False, cascade_cls=False, use_depth_gt=True),
    "kitti_b3_f32_flospdepth_2080ti": dict(   # semantic_kitti/multicam_flospdepth_crp_stereodepth_cascadecls_2080ti
        dataset="kitti", backbone_2d_name="tf_efficientnet_b3_ns", feature=32, trans_2d_to_3d="flosp_depth", views=2,
        context_prior=True, cascade_cls=True, use_stereo_depth_gt=True),   # (released KITTI model)
    "kitti_b3_f24_flospdepth_mono_2080ti": dict(   # semantic_kitti/flospdepth_2080ti.yaml (multi_view_mode: false)
        dataset="kitti", backbone_2d_name="tf_efficientnet_b3_ns", feature=24, trans_2d_to_3d="flosp_depth", views=1,
        context_prior=False, cascade_cls=False, multi_view_mode=False),
    "kitti_b7_f64_flosp_a100": dict(   # semantic_kitti/multicam_flosp_crp_cascadecls_a100.yaml
        dataset="kitti", backbone_2d_name="tf_efficientnet_b7_ns", feature=64, trans_2d_to_3d="flosp", views=2,
        context_prior=True, cascade_cls=True),
    "kitti_b7_f64_flospdepth_a100": dict(   # semantic_kitti/multicam_flospdepth_crp_stereodepth_cascadecls_a100.yaml
        dataset="kitti", backbone_2d_name="tf_efficientnet_b7_ns", feature=64, trans_2d_to_3d="flosp_depth", views=2,
        context_prior=True, cascade_cls=True, use_stereo_depth_gt=True),
    "nyu_b7_f200_v100": dict(   # NYU/multicam_flospdepth_crp_stereodepth_cascadecls_v100.yaml
        dataset="NYU", backbone_2d_name="tf_efficientnet_b7_ns", feature=200, trans_2d_to_3d="flosp", views=1,
        context_prior=True, cascade_cls=False, use_depth_gt=True),
}


def make_case(name=None, spec=None, img_hw=None, full=None, seed=0, infer_mode=False):
    """-> (model (CPU, eval), batch (CPU tensors), oracle cfg) for CONFIGS[name] (or an explicit spec) at the shipped
    shapes, or at img_hw / full when given.  KITTI views use KITTI-like calibrations; NYU takes one image and a depth
    map (virtual stereo) with seeded random projection indices.  infer_mode builds the model for the reference's
    deployment route (OccDepth(infer_mode=True)); the batch then still carries camera matrices, not grids."""
    import torch
    import synthetic as synth
    from occdepth_b200.models.OccDepth import OccDepth
    import occdepth_b200.models.flosp_depth.flosp_depth as fd
    spec = dict(CONFIGS[name] if spec is None else spec)
    ds, V, f = spec.pop("dataset"), spec.pop("views"), spec.pop("feature")
    nyu = ds == "NYU"
    H, W = img_hw or (NYU_IMG if nyu else KITTI_IMG)
    full = tuple(full or (NYU_FULL if nyu else KITTI_FULL))
    ps = 1 if nyu else 2
    ncls = 12 if nyu else 20
    cfg = synth.occdepth_cfg(dataset=ds, full_scene_size=full, project_scale=ps, feature=f, feature_2d_oc=f,
                             n_classes=ncls, **spec)
    conf_saved = copy.deepcopy(fd.flosp_depth_conf_map[ds])
    try:
        if cfg.trans_2d_to_3d == "flosp_depth" and not nyu:
            # the frustum of the image actually fed; a smaller scene keeps the 0.2 m voxels from the same corner
            fd.flosp_depth_conf_map[ds].update(final_dim=(H, W))
            if full != KITTI_FULL:
                sm = [s * 0.2 for s in full]
                fd.flosp_depth_conf_map[ds].update(x_bound=[0, sm[0], 0.2], y_bound=[-sm[1] / 2, sm[1] / 2, 0.2],
                                                   z_bound=[-2, -2 + sm[2], 0.2])
        torch.manual_seed(seed)
        with contextlib.redirect_stdout(io.StringIO()):
            m = OccDepth(["c"] * ncls, torch.ones(ncls), full_scene_size=full, project_res=PROJECT_RES, config=cfg,
                         infer_mode=infer_mode)
        conf = copy.deepcopy(getattr(m, "flosp_depth_conf", None))
    finally:
        fd.flosp_depth_conf_map[ds].clear()
        fd.flosp_depth_conf_map[ds].update(conf_saved)
    if conf is not None:
        m.flosp_depth_conf = copy.deepcopy(conf)     # the model held the shared default dict, restored just above
    synth.randomize_bn_(m)
    m = m.eval()
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(1, V, 3, H, W, generator=g)
    N = (full[0] // ps) * (full[1] // ps) * (full[2] // ps)
    if nyu:
        depth = torch.rand(1, 1, H, W, generator=g) * 7.5 + 0.5
        pix, fov = synth.random_indices(N, W, H, n_views=2, P=1, seed=seed + 1, margin=(W // 4, H // 4))
        batch = {"img": img, "gt_depth": depth, "virtual_bf": [torch.tensor(51.88579)],
                 "vox_origin": torch.zeros(1, 3, dtype=torch.float64), "projected_pix_1": [pix], "fov_mask_1": [fov]}
    else:
        pix, fov, K, Ts = synth.kitti_indices(W, H, full, ps, voxel=0.2, n_views=V)
        batch = {"img": img, "projected_pix_2": [pix], "fov_mask_2": [fov]}
        if cfg.trans_2d_to_3d == "flosp_depth":
            batch.update(cam_k=[torch.from_numpy(K).unsqueeze(0).repeat(V, 1, 1)],
                         T_velo_2_cam=[torch.stack([torch.from_numpy(t) for t in Ts[:V]])],
                         ida_mats=[torch.eye(4).unsqueeze(0).repeat(V, 1, 1)])
    ocfg = dict(cfg)
    ocfg.update(project_res=PROJECT_RES, flosp_depth_conf=conf, with_depth_gt=m.with_depth_gt)
    return m, batch, ocfg


DEVICE_KEYS = ("img", "gt_depth", "projected_pix_", "fov_mask_")


def to_cuda(batch):
    """the image, the depth map and the per-frame projection indices / FOV masks on the device; the camera matrices,
    `vox_origin` and `virtual_bf` are read on the host by the forward and stay there"""
    b = dict(batch)
    for k, v in batch.items():
        if k.startswith(DEVICE_KEYS):
            b[k] = [t.cuda() for t in v] if isinstance(v, list) else v.cuda()
    return b


def card():
    """name and power limit of the current device; nvidia-smi is asked by UUID, since its indices need not match
    torch's under CUDA_VISIBLE_DEVICES"""
    import torch
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", "GPU-%s" % props.uuid], capture_output=True, text=True,
                            timeout=30).stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return props.name, pl


def time_forward(m, batch, steps, warmup, repeats=1):
    """ms per forward of `repeats` windows of `steps` forwards each, after `warmup` forwards"""
    import torch
    res = []
    with torch.no_grad():
        for _ in range(warmup):
            m(batch)
        for _ in range(repeats):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                m(batch)
            e1.record()
            torch.cuda.synchronize()
            res.append(e0.elapsed_time(e1) / steps)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("shipped_configs.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = card()
    for name in a.names:
        m, batch, _ = make_case(name)
        m = m.cuda()
        b = to_cuda(batch)
        spec = CONFIGS[name]
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            ms = time_forward(m, b, a.steps, a.warmup, a.repeats)
            print(json.dumps(dict(config=name, precision=prec, ms_per_frame=round(statistics.median(ms), 3),
                                  windows_ms=[round(t, 3) for t in ms],
                                  backbone=spec["backbone_2d_name"], feature=spec["feature"],
                                  trans_2d_to_3d=spec["trans_2d_to_3d"], views=spec["views"], steps=a.steps,
                                  warmup=a.warmup, gpu=gpu, power_limit=power)), flush=True)
        del m, b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
