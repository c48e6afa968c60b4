"""BASELINE.json configs[3]: NYUv2-shape 640x480 RGB-D (virtual stereo), EfficientNet-B7, 60x36x60 / 200-channel
grid, NYU 3-D UNet with CRP -- the dense small-grid / high-channel path (C = 200 lift, 200/400/800-channel 3-D convs,
196-position mega-context).  CUDA forward vs the CPU fp32 oracle on the same seeded inputs and weights."""
import contextlib
import io

import pytest
import torch

import gpu_cases as G

pytestmark = pytest.mark.gpu
# about 2x the values measured; see tests/test_gpu_config2.py.  Measured on an H100 SXM (700 W): tf32 rel 8.9e-4,
# P_logits 5.6e-4, arg-max 99.951 %; bf16 rel 6.3e-3, P_logits 4.4e-3, arg-max 99.687 %
TOL = {"tf32": dict(rel=1.6e-3, argmax=0.9991), "bf16": dict(rel=1.25e-2, argmax=0.9935)}


@pytest.fixture(scope="module")
def case():
    import synthetic as synth
    from oracle import functional as OF
    from occdepth_b200.models.OccDepth import OccDepth
    torch.manual_seed(0)
    full = (60, 36, 60)
    H, W = 480, 640
    cfg = synth.occdepth_cfg(dataset="NYU", full_scene_size=full, project_scale=1, feature=200, feature_2d_oc=200,
                             n_classes=12, cascade_cls=False, context_prior=True,
                             backbone_2d_name="tf_efficientnet_b7_ns")
    with contextlib.redirect_stdout(io.StringIO()):
        m = OccDepth(["c"] * 12, torch.ones(12), full_scene_size=full, project_res=["1", "2", "4", "8"], config=cfg)
    synth.randomize_bn_(m)
    m = m.eval()
    g = torch.Generator().manual_seed(0)
    img = torch.randn(1, 1, 3, H, W, generator=g)
    depth = torch.rand(1, 1, H, W, generator=g) * 7.5 + 0.5
    N = full[0] * full[1] * full[2]
    pix, fov = synth.random_indices(N, W, H, n_views=2, P=1, seed=1, margin=(160, 120))   # FOV fraction ~0.44
    batch = {"img": img, "gt_depth": depth, "virtual_bf": [torch.tensor(51.88579)],
             "vox_origin": torch.zeros(1, 3, dtype=torch.float64), "projected_pix_1": [pix], "fov_mask_1": [fov]}
    ocfg = dict(cfg)
    ocfg["project_res"] = ["1", "2", "4", "8"]
    with torch.no_grad():
        want = OF.occdepth_forward({k: v.clone() for k, v in m.state_dict().items()}, batch, ocfg)
    b2 = dict(batch)
    b2["img"] = img.cuda()
    return m.cuda(), b2, want, N


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_config4_logits_vs_oracle(case, precision):
    m, b2, want, N = case
    m.set_precision(precision)
    with torch.no_grad():
        got = m(b2)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            m(b2)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    g_, w_ = got["ssc_logit"].float().cpu(), want["ssc_logit"]
    rep = {"precision": precision, "max_abs_diff": float((g_ - w_).abs().max()), "max_abs_ref": float(w_.abs().max()),
           "rel": float((g_ - w_).abs().max() / w_.abs().max()),
           "argmax_agreement": float((g_.argmax(1) == w_.argmax(1)).float().mean()),
           "P_logits_rel": float((got["P_logits"].cpu() - want["P_logits"]).abs().max() / want["P_logits"].abs().max()),
           "ms_per_frame": ms, "voxels_per_s": N / ms * 1e3}
    G.write_report("config4_parity_%s.json" % precision, rep)
    print("config-4 parity:", rep)
    t = TOL[precision]
    assert rep["rel"] <= t["rel"] and rep["P_logits_rel"] <= t["rel"], rep
    assert rep["argmax_agreement"] >= t["argmax"], rep
