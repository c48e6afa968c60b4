"""Import the UNMODIFIED reference (`$OCCDEPTH_REFERENCE/occdepth`, a checkout of the original project) as the
ground-truth oracle.

Only possible where that checkout exists; oracle/gen_golden.py stores what the tests compare against, so the test
suite itself never needs it.  Third-party imports missing
from this image are satisfied by `oracle/shims/` (see its README) and `torch.hub.load` is redirected to the
geffnet-shaped EfficientNet of `oracle/effnet.py` (random init -- no network for pretrained weights).
"""
import contextlib
import io
import os
import sys
import types

REF_ROOT = os.environ.get("OCCDEPTH_REFERENCE", "")
_SHIMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shims")


def available():
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "occdepth", "models"))


def _install():
    if not available():
        raise RuntimeError("reference tree not found (set OCCDEPTH_REFERENCE to a checkout of the original project)")
    for p in (_SHIMS, REF_ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch
    from . import effnet

    if not getattr(torch.hub, "_occd_patched", False):
        orig = torch.hub.load

        def load(repo, model, *a, **k):
            if "gen-efficientnet-pytorch" in str(repo):
                return effnet.GenEfficientNet(model)
            return orig(repo, model, *a, **k)

        torch.hub.load = load
        torch.hub._occd_patched = True


def modules():
    """Returns a namespace with the reference's hot-path modules (imported quietly)."""
    _install()
    ns = types.SimpleNamespace()
    with contextlib.redirect_stdout(io.StringIO()):
        import occdepth.models.SFA as SFA
        import occdepth.models.DDR as DDR
        import occdepth.models.modules as mods
        import occdepth.models.CRP3D as CRP3D
        import occdepth.models.unet3d_kitti as unet3d_kitti
        import occdepth.models.unet3d_nyu as unet3d_nyu
        import occdepth.models.unet2d as unet2d
        import occdepth.models.OccDepth as OccDepth
        import occdepth.models.flosp_depth.flosp_depth as flosp_depth
    ns.SFA, ns.DDR, ns.modules, ns.CRP3D = SFA, DDR, mods, CRP3D
    ns.unet3d_kitti, ns.unet3d_nyu, ns.unet2d = unet3d_kitti, unet3d_nyu, unet2d
    ns.OccDepth, ns.flosp_depth = OccDepth, flosp_depth
    return ns


def data_helpers():
    """The reference's projection helpers (occdepth/data/utils/helpers.py, numba-compiled fusion.py); needs numba,
    and the `skimage` shim for an import on the mesh-export path that the projection never touches."""
    _install()
    import warnings
    with contextlib.redirect_stdout(io.StringIO()), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        import occdepth.data.utils.helpers as helpers
    return helpers


@contextlib.contextmanager
def quiet():
    with contextlib.redirect_stdout(io.StringIO()):
        yield
