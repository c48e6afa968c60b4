"""3D network drop-in modules on CUDA vs the CPU fp32 oracle (same seeded weights)."""
import pytest
import torch
import torch.nn as nn

from oracle import functional as OF
from oracle import synth

import gpu_cases as G

pytestmark = pytest.mark.gpu
PREC = pytest.mark.parametrize("precision", G.PRECISIONS)

# stated tolerance on max-abs-diff relative to max-abs of the oracle tensor, per precision mode (about 2x the values
# measured; OCCDEPTH_PARITY_DIR=<dir> records them); ~25 fused layers between input and logits
TOL = {"tf32": 1.5e-3, "bf16": 1.4e-2}
TOL_BLOCK = {"tf32": 1.5e-3, "bf16": 1.5e-2}
TOL_ARGMAX = {"tf32": 0.9995, "bf16": 0.99}


def _check(name, precision, got, want, tol):
    errs = {}
    for k in want:
        g, w = got[k].float().cpu(), want[k]
        assert g.shape == w.shape, (k, g.shape, w.shape)
        errs[k] = float((g - w).abs().max() / w.abs().max().clamp_min(1e-6))
    G.record(name, precision, **errs)
    for k, err in errs.items():
        assert err <= tol, (k, err)


@PREC
def test_process_downsample_upsample(precision):
    from occdepth_b200.models.modules import Downsample, Process, Upsample
    torch.manual_seed(0)
    proc = Process(32, nn.BatchNorm3d, 0.1).eval()
    down = Downsample(32, nn.BatchNorm3d, 0.1).eval()
    up = Upsample(64, 32, nn.BatchNorm3d, 0.1).eval()
    for m in (proc, down, up):
        synth.randomize_bn_(m)
    x = torch.randn(1, 32, 12, 10, 8)
    with torch.no_grad():
        want_p = OF.process({"p." + k: v for k, v in proc.state_dict().items()}, "p", x)
        want_d = OF.downsample({"p." + k: v for k, v in down.state_dict().items()}, "p", x)
        want_u = OF.upsample({"p." + k: v for k, v in up.state_dict().items()}, "p", want_d)
        t = TOL_BLOCK[precision]
        _check("process", precision, {"p": proc.cuda().set_precision(precision)(x.cuda())}, {"p": want_p}, t)
        _check("downsample", precision, {"d": down.cuda().set_precision(precision)(x.cuda())}, {"d": want_d}, t)
        _check("upsample", precision, {"u": up.cuda().set_precision(precision)(want_d.cuda())}, {"u": want_u}, t)


@PREC
@pytest.mark.parametrize("which", ["kitti", "nyu"])
def test_unet3d(which, precision):
    torch.manual_seed(0)
    if which == "kitti":
        from occdepth_b200.models.unet3d_kitti import UNet3D
        full, ps, f = (32, 32, 16), 2, 32
        m = UNet3D(20, nn.BatchNorm3d, full, f, ps, context_prior=True, cascade_cls=True, occluded_cls=True).eval()
        x = torch.randn(1, f, 16, 16, 8)
    else:
        from occdepth_b200.models.unet3d_nyu import UNet3D
        full, f = (12, 8, 12), 24
        m = UNet3D(12, nn.BatchNorm3d, f, full, context_prior=True, cascade_cls=False).eval()
        x = torch.randn(1, f, 12, 8, 12)
    synth.randomize_bn_(m)
    sd = {"n." + k: v.clone() for k, v in m.state_dict().items()}
    with torch.no_grad():
        if which == "kitti":
            want = OF.unet3d_kitti(sd, "n", x, full, ps, True, True, True)
        else:
            want = OF.unet3d_nyu(sd, "n", x, full, 4, True, False)
        got = m.cuda().set_precision(precision)({"x3d": x.cuda()})
    assert set(got.keys()) == set(want.keys())
    agree = float((got["ssc_logit"].argmax(1).cpu() == want["ssc_logit"].argmax(1)).float().mean())
    G.record("unet3d[%s].argmax" % which, precision, argmax=agree)
    _check("unet3d[%s]" % which, precision, got, want, TOL[precision])
    assert agree >= TOL_ARGMAX[precision], agree
