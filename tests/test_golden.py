"""Oracle (oracle/functional.py) vs the committed golden vectors produced by the UNMODIFIED reference
(oracle/gen_golden.py).  Runs anywhere (CPU); with tests/test_oracle_vs_reference.py this is what pins the oracle."""
import os

import torch
import torch.nn as nn

from oracle import functional as OF
from oracle import synth

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _close(a, b, rtol=1e-3, atol=1e-4):
    assert a.shape == b.shape
    assert torch.allclose(a, b, rtol=rtol, atol=atol), float((a - b).abs().max())


def test_sfa_golden():
    d = torch.load(os.path.join(G, "sfa.pt"))
    assert len(d) == 5
    for c in d.values():
        _close(OF.sfa(c["x2d"], c["pix"], c["fov"], c["scene"], c["dataset"], c["ps"]), c["out"], 1e-5, 1e-6)


def _product_module(which):
    # the CUDA package's modules are used here ONLY as parameter containers (identical state_dict keys)
    if which == "kitti":
        from occdepth_b200.models.unet3d_kitti import UNet3D
        return UNet3D(5, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=True, cascade_cls=True,
                      occluded_cls=True)
    from occdepth_b200.models.unet3d_nyu import UNet3D
    return UNet3D(5, nn.BatchNorm3d, 16, (12, 8, 12), context_prior=True, cascade_cls=False)


def test_unet3d_golden(capsys):
    d = torch.load(os.path.join(G, "unet3d.pt"))
    for which in ("kitti", "nyu"):
        c = d[which]
        m = synth.seed_weights_(_product_module(which), c["seed"])
        sd = {"n." + k: v for k, v in m.state_dict().items()}
        with torch.no_grad():
            if which == "kitti":
                got = OF.unet3d_kitti(sd, "n", c["x"], (32, 32, 16), 2, True, True, True)
            else:
                got = OF.unet3d_nyu(sd, "n", c["x"], (12, 8, 12), 4, True, False)
        for k, v in c["out"].items():
            _close(got[k], v)


def test_occdepth_golden():
    c = torch.load(os.path.join(G, "occdepth_small.pt"))
    from occdepth_b200.models.OccDepth import OccDepth
    cfg = synth.Cfg(c["cfg"])
    m = OccDepth(["c"] * 6, torch.ones(6), full_scene_size=(32, 32, 16), project_res=["1", "2", "4", "8"], config=cfg)
    synth.seed_weights_(m, c["seed"])
    ocfg = dict(cfg)
    ocfg["project_res"] = ["1", "2", "4", "8"]
    batch = {"img": c["img"], "projected_pix_2": [c["pix"]], "fov_mask_2": [c["fov"]]}
    with torch.no_grad():
        got = OF.occdepth_forward(m.state_dict(), batch, ocfg)
        feats = OF.unet2d(m.state_dict(), "net_rgb", c["img"][:, 0], cfg.backbone_2d_name, 1)
    _close(got["ssc_logit"], c["ssc_logit"], 2e-3, 2e-4)
    _close(got["occ_logit"], c["occ_logit"], 2e-3, 2e-4)
    _close(feats["1_8"], c["feat_1_8"], 2e-3, 2e-4)
