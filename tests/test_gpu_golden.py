"""CUDA path vs the committed golden vectors of the UNMODIFIED reference (tests/golden/, oracle/gen_golden.py)."""
import os

import pytest
import torch
import torch.nn as nn

from oracle import synth

import gpu_cases as GC

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PREC = pytest.mark.parametrize("precision", GC.PRECISIONS)
# relative to max-abs of the reference's tensor, per precision mode (about 2x the values measured)
# measured: 3-D nets tf32 <= 2.2e-3 (P_logits, |max| 9) / bf16 <= 1.05e-2; full forward tf32 7.0e-4 / bf16 6.8e-3
TOL_3D = {"tf32": 4e-3, "bf16": 2e-2}
TOL_E2E = {"tf32": 1.4e-3, "bf16": 1.4e-2}


def _rel(g, w):
    return float((g.float().cpu() - w).abs().max() / w.abs().max().clamp_min(1e-6))


def test_sfa_golden_gpu():
    from occdepth_b200.models.SFA import SFA
    d = torch.load(os.path.join(G, "sfa.pt"))
    for c in d.values():
        got = SFA(c["scene"], c["dataset"], c["ps"])(c["x2d"].cuda(), c["pix"].cuda(), c["fov"].cuda()).cpu()
        assert float((got - c["out"]).abs().max()) <= 1e-5


@PREC
def test_unet3d_golden_gpu(precision):
    from test_golden import _product_module
    d = torch.load(os.path.join(G, "unet3d.pt"))
    for which in ("kitti", "nyu"):
        c = d[which]
        m = synth.seed_weights_(_product_module(which), c["seed"]).eval().cuda().set_precision(precision)
        with torch.no_grad():
            got = m({"x3d": c["x"].cuda()})
        GC.record("unet3d_golden[%s]" % which, precision, **{k: _rel(got[k], v) for k, v in c["out"].items()})
        for k, v in c["out"].items():
            assert _rel(got[k], v) <= TOL_3D[precision], (which, k, _rel(got[k], v))


@PREC
def test_occdepth_golden_gpu(precision):
    from occdepth_b200.models.OccDepth import OccDepth
    c = torch.load(os.path.join(G, "occdepth_small.pt"))
    cfg = synth.Cfg(c["cfg"])
    m = OccDepth(["c"] * 6, torch.ones(6), full_scene_size=(32, 32, 16), project_res=["1", "2", "4", "8"], config=cfg)
    synth.seed_weights_(m, c["seed"])
    m = m.eval().cuda().set_precision(precision)
    with torch.no_grad():
        got = m({"img": c["img"].cuda(), "projected_pix_2": [c["pix"]], "fov_mask_2": [c["fov"]]})
    GC.record("occdepth_golden", precision, **{k: _rel(got[k], c[k]) for k in ("ssc_logit", "occ_logit")})
    for k in ("ssc_logit", "occ_logit"):
        assert _rel(got[k], c[k]) <= TOL_E2E[precision], (k, _rel(got[k], c[k]))
