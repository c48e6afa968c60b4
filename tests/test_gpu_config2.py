"""Full-size parity at the benchmark configuration (BASELINE.json configs[1]): CUDA forward vs the CPU fp32 oracle
on the same seeded stereo pair / weights / KITTI-like projection indices, in both precision modes.  The metric the north
star names: voxel-logit max-abs-diff (also reported relative to max |logit|) plus arg-max agreement."""

import pytest
import torch

import gpu_cases as G

pytestmark = pytest.mark.gpu

# stated tolerances (about 2x the values measured): relative = max-abs-diff /
# max |oracle logit|.  tf32 = the reference-precision mode (TF32 operands, fp32 accumulation, TF32-valued fp32
# activations); bf16 = the throughput mode.  A CPU simulation of the tf32 mode (TF32-rounded conv operands inside the
# fp32 oracle) gives rel 6.3e-4 / arg-max 99.93 %, so these bounds are what the arithmetic allows, not slack for bugs.
# measured on an H100 SXM (700 W): tf32 rel 6.3e-4 (ssc) / 7.7e-4 (occ), arg-max 99.927 %; bf16 rel 6.3e-3 / 8.2e-3,
# arg-max 99.194 %
TOL = {"tf32": dict(rel=1.5e-3, argmax=0.9984), "bf16": dict(rel=1.4e-2, argmax=0.984)}


@pytest.fixture(scope="module")
def case():
    import bench
    from oracle import functional as OF
    m = bench.build_model()
    img, pix, fov = bench.make_inputs(seed=0)
    cfg = dict(bench.make_cfg())
    cfg["project_res"] = bench.PROJECT_RES
    batch = {"img": img, "projected_pix_2": [pix], "fov_mask_2": [fov]}
    with torch.no_grad():
        want = OF.occdepth_forward({k: v.clone() for k, v in m.state_dict().items()}, batch, cfg)
    return m.cuda(), {"img": img.cuda(), "projected_pix_2": [pix], "fov_mask_2": [fov]}, want


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_config2_logits_vs_oracle(case, precision):
    m, batch, want = case
    with torch.no_grad():
        got = m.set_precision(precision)(batch)
    rep = {"precision": precision}
    for k in ("ssc_logit", "occ_logit"):
        g, w = got[k].float().cpu(), want[k]
        assert g.shape == w.shape
        rep[k] = {"max_abs_diff": float((g - w).abs().max()), "max_abs_ref": float(w.abs().max()),
                  "rel": float((g - w).abs().max() / w.abs().max())}
    agree = float((got["ssc_logit"].argmax(1).cpu() == want["ssc_logit"].argmax(1)).float().mean())
    rep["argmax_agreement"] = agree
    G.write_report("config2_parity_%s.json" % precision, rep)
    print("config-2 parity:", rep)
    t = TOL[precision]
    assert rep["ssc_logit"]["rel"] <= t["rel"] and rep["occ_logit"]["rel"] <= t["rel"], rep
    assert agree >= t["argmax"], rep


# ---- the config-2 "extended variant" (SURVEY 8d): trans_2d_to_3d = "flosp_depth" as in
# multicam_flospdepth_crp_stereodepth_cascadecls_a100.yaml with final_dim = (376, 1370): DepthNet over both views' 1/8
# maps (47 x 172), 104 depth bins, frustum sampling to the 128 x 128 x 16 grid, prior x lift x 100 ----
# measured on an H100 SXM (700 W): tf32 rel <= 9.9e-4; bf16 <= 8.5e-3
TOL_FD = {"tf32": dict(rel=2.1e-3, argmax=0.9987), "bf16": dict(rel=1.7e-2, argmax=0.9825)}


@pytest.fixture(scope="module")
def case_flosp_depth():
    import contextlib
    import copy
    import io
    import bench
    import synthetic as synth
    from oracle import functional as OF
    from occdepth_b200.models.OccDepth import OccDepth
    import occdepth_b200.models.flosp_depth.flosp_depth as fd
    H, W = bench.IMG_H, bench.IMG_W
    saved = copy.deepcopy(fd.flosp_depth_conf_map["kitti"])
    try:
        fd.flosp_depth_conf_map["kitti"].update(final_dim=(H, W))
        cfg = synth.occdepth_cfg(full_scene_size=bench.FULL, project_scale=2, feature=64, feature_2d_oc=64, n_classes=20,
                                 backbone_2d_name="tf_efficientnet_b7_ns", cascade_cls=True, context_prior=True,
                                 trans_2d_to_3d="flosp_depth", use_stereo_depth_gt=True)
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            m = OccDepth(["c"] * 20, torch.ones(20), full_scene_size=bench.FULL, project_res=bench.PROJECT_RES,
                         config=cfg)
        conf = copy.deepcopy(m.flosp_depth_conf)
    finally:
        fd.flosp_depth_conf_map["kitti"].clear()
        fd.flosp_depth_conf_map["kitti"].update(saved)
    synth.randomize_bn_(m)
    m = m.eval()
    img, pix, fov = bench.make_inputs(seed=0)
    K, Ts = synth.kitti_calib(W, H)
    batch = {"img": img, "projected_pix_2": [pix], "fov_mask_2": [fov],
             "cam_k": [torch.from_numpy(K).unsqueeze(0).repeat(2, 1, 1)],
             "T_velo_2_cam": [torch.stack([torch.from_numpy(t) for t in Ts])],
             "ida_mats": [torch.eye(4).unsqueeze(0).repeat(2, 1, 1)]}
    ocfg = dict(cfg)
    ocfg.update(project_res=bench.PROJECT_RES, flosp_depth_conf=conf, with_depth_gt=True)
    with torch.no_grad():
        want = OF.occdepth_forward({k: v.clone() for k, v in m.state_dict().items()}, batch, ocfg)
    b2 = dict(batch)
    b2["img"] = img.cuda()
    return m.cuda(), b2, want


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_config2_flosp_depth_vs_oracle(case_flosp_depth, precision):
    m, batch, want = case_flosp_depth
    with torch.no_grad():
        got = m.set_precision(precision)(batch)
    rep = {"precision": precision, "depth_pred_shape": list(got["depth_pred"].shape)}
    assert tuple(got["depth_pred"].shape) == tuple(want["depth_pred"].shape) == (1, 2, 104, 47, 172)
    for k in ("ssc_logit", "occ_logit", "depth_pred"):
        g, w = got[k].float().cpu(), want[k]
        rep[k] = {"max_abs_diff": float((g - w).abs().max()), "max_abs_ref": float(w.abs().max()),
                  "rel": float((g - w).abs().max() / w.abs().max())}
    agree = float((got["ssc_logit"].argmax(1).cpu() == want["ssc_logit"].argmax(1)).float().mean())
    rep["argmax_agreement"] = agree
    G.write_report("config2_flospdepth_parity_%s.json" % precision, rep)
    print("config-2 (flosp_depth) parity:", rep)
    t = TOL_FD[precision]
    assert all(rep[k]["rel"] <= t["rel"] for k in ("ssc_logit", "occ_logit", "depth_pred")), rep
    assert agree >= t["argmax"], rep
