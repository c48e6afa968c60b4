"""Pins oracle/functional.py against the UNMODIFIED reference modules (CPU fp32, seeded weights).

The reference's outputs are stored in tests/golden/reference_pins.pt (oracle/gen_golden.py, run where the original
project is importable); the inputs are regenerated from the same seeds.  Weights are synth.seed_weights_ fills, which
the CUDA package's modules reproduce (identical state_dict keys); they serve here ONLY as parameter containers.
"""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import functional as OF
from oracle import gen_golden, projection, synth

PINS = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins.pt"),
                  weights_only=False)
TOL = dict(rtol=1e-4, atol=1e-5)


def _close(a, b, **kw):
    """b: a stored reference tensor, or {shape, values}: the reference's values at gen_golden.pin_index"""
    tol = dict(TOL)
    tol.update(kw)
    if isinstance(b, dict):
        assert tuple(a.shape) == tuple(b["shape"]), (a.shape, b["shape"])
        a, b = a.contiguous().reshape(-1)[gen_golden.pin_index(a.numel())], b["values"]
    assert a.shape == b.shape, (a.shape, b.shape)
    assert torch.allclose(a, b, **tol), float((a - b).abs().max())


@pytest.mark.parametrize("dataset,V,P", gen_golden.SFA_CASES)
def test_sfa(dataset, V, P):
    x2d, pix, fov = gen_golden.sfa_pin_inputs(V, P)
    got = OF.sfa(x2d, pix, fov, (16, 12, 8), dataset, 2)
    _close(got, PINS["sfa_%s_%d_%d" % (dataset, V, P)], rtol=1e-5, atol=1e-6)


def test_bottleneck_process_downsample():
    from occdepth_b200.models import modules
    c = PINS["blocks"]
    x = gen_golden.blocks_pin_input()
    sds = []
    for i, m in enumerate(gen_golden.block_modules(types.SimpleNamespace(modules=modules))):
        sds.append({"p." + k: v for k, v in synth.seed_weights_(m, 40 + i).state_dict().items()})
    with torch.no_grad():
        _close(OF.process(sds[0], "p", x), c["process"])
        y = OF.downsample(sds[1], "p", x)
        _close(y, c["downsample"])
        _close(OF.upsample(sds[2], "p", y), c["upsample"])


@pytest.mark.parametrize("which", ["kitti", "nyu"])
def test_unet3d(which):
    xk, xn = gen_golden.unet3d_pin_inputs()
    if which == "kitti":
        from occdepth_b200.models.unet3d_kitti import UNet3D
        full, ps, x, seed = (32, 32, 16), 2, xk, 31
        m = UNet3D(5, nn.BatchNorm3d, full, 16, ps, context_prior=True, cascade_cls=True, occluded_cls=True)
    else:
        from occdepth_b200.models.unet3d_nyu import UNet3D
        full, x, seed = (12, 8, 12), xn, 32
        m = UNet3D(5, nn.BatchNorm3d, 16, full, context_prior=True, cascade_cls=False)
    sd = {"n." + k: v for k, v in synth.seed_weights_(m, seed).state_dict().items()}
    want = PINS["unet3d_" + which]
    with torch.no_grad():
        if which == "kitti":
            got = OF.unet3d_kitti(sd, "n", x, full, ps, True, True, True)
        else:
            got = OF.unet3d_nyu(sd, "n", x, full, 4, True, False)
    assert set(got.keys()) == set(want.keys())
    for k in want:
        _close(got[k], want[k], rtol=1e-3, atol=1e-4)


def test_unet2d():
    from occdepth_b200.models.unet2d import UNet2D
    m = UNet2D.build(out_feature=16, use_decoder=True, backbone_2d_name="tf_efficientnet_b3_ns", return_up_feats=1)
    sd = {"net_rgb." + k: v for k, v in synth.seed_weights_(m, 33).state_dict().items()}
    want = PINS["unet2d"]
    with torch.no_grad():
        got = OF.unet2d(sd, "net_rgb", gen_golden.unet2d_pin_input(), "tf_efficientnet_b3_ns", 1)
    assert set(got.keys()) == set(want.keys())
    for k in want:
        _close(got[k], want[k], rtol=1e-3, atol=1e-4)


def _occdepth(full, cfg, batch, seed, want):
    from occdepth_b200.models.OccDepth import OccDepth
    m = OccDepth(["c"] * 6, torch.ones(6), full_scene_size=full, project_res=["1", "2", "4", "8"], config=cfg)
    synth.seed_weights_(m, seed)
    ocfg = dict(cfg)
    ocfg["project_res"] = ["1", "2", "4", "8"]
    with torch.no_grad():
        got = OF.occdepth_forward(m.state_dict(), batch, ocfg)
    assert set(got.keys()) == set(want.keys())
    for k in want:
        _close(got[k], want[k], rtol=2e-3, atol=2e-4)


def test_occdepth_forward_small():
    """whole OccDepth.forward ("flosp", kitti decoder with CRP + cascade) on a tiny stereo pair."""
    _occdepth(*gen_golden.occdepth_small_pin_inputs(), 34, PINS["occdepth_small"])


def test_flosp_depth():
    """FlospDepth (DepthNet + frustum grid + trilinear sampling + masked mean), kitti geometry, 2 cameras"""
    from occdepth_b200.models.flosp_depth import FlospDepth, flosp_depth_conf_map
    c = PINS["flosp_depth"]
    conf, feat, cam_k, T, ida = gen_golden.flosp_pin_inputs(flosp_depth_conf_map)
    m = synth.seed_weights_(FlospDepth(**conf), 5)
    with torch.no_grad():
        got, got_d = OF.flosp_depth({"f." + k: v for k, v in m.state_dict().items()}, "f", feat, cam_k, T, ida, conf)
    assert c["cover"] > 0.2     # the frustum actually covers part of the grid
    _close(got_d, c["depth"], rtol=1e-4, atol=1e-6)
    _close(got, c["out"], rtol=1e-3, atol=1e-5)


def _nyu_virtual_batch(H, W, full, seed=0):
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(1, 1, 3, H, W, generator=g)
    depth = torch.rand(1, 1, H, W, generator=g) * 7.5 + 0.5
    depth[0, 0, 3, 5] = 0.0          # exercises the inf -> 0 disparity rule (OccDepth.py:248)
    N = full[0] * full[1] * full[2]
    pix, fov = synth.random_indices(N, W, H, n_views=2, P=1, seed=seed + 1, margin=(8, 6))
    return {"img": img, "gt_depth": depth, "virtual_bf": [torch.tensor(51.88579 * W / 640.0)],
            "vox_origin": torch.zeros(1, 3, dtype=torch.float64), "projected_pix_1": [pix], "fov_mask_1": [fov]}


def test_occdepth_forward_nyu_virtual_view():
    """NYU-type path: one real view, the right view synthesised from gt_depth (generate_virtual_img)"""
    _occdepth(*gen_golden.nyu_virtual_pin_inputs(), 3, PINS["occdepth_nyu_virtual_view"])


@pytest.mark.parametrize("pattern_id", [0, 1, 3, 6, 8])
def test_vox2pix_against_the_numba_reference(pattern_id):
    """oracle/projection.py vs occdepth.data.utils.helpers.vox2pix itself (numba-compiled), bit for bit: dtype,
    shape and a digest of the bytes of every output"""
    dig = PINS["vox2pix_digests"]
    for name, E, K, org, vs, W, H, scene, _ in gen_golden.vox2pix_cases():
        got = projection.vox2pix(E, K, org, vs, W, H, scene, pattern_id)
        assert [gen_golden.pin_digest(np.asarray(g)) for g in got] == dig["%s_%d" % (name, pattern_id)], name
