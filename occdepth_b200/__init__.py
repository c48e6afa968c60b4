"""occdepth_b200 -- H100 (sm_90a) native forward hot path of OccDepth.

Module surface mirrors the reference's `occdepth.models` (same class names, constructor signatures, forward
inputs/outputs and state_dict keys); `install_as_occdepth()` registers this package under the reference's
import names so its train/eval scripts import it unchanged (see INTEGRATION.md).
"""
__version__ = "0.1.0"


def install_as_occdepth():
    """Expose occdepth_b200.models.* as occdepth.models.* (the reference's import paths).

    `occdepth` itself stays a real package: when the reference tree is importable (on sys.path) its namespace package
    is kept, so `occdepth.data.*`, `occdepth.loss.*` and `occdepth.scripts.*` keep resolving to the reference while
    `occdepth.models` and its hot-path submodules resolve to this package.  Without the reference on the path a
    package stub (with an empty `__path__`) is registered, so imports of anything but `occdepth.models*` fail with an
    ordinary ModuleNotFoundError.  Call it BEFORE the first `import occdepth.models...`."""
    import importlib
    import importlib.util
    import sys
    import types

    names = ["SFA", "DDR", "modules", "CRP3D", "unet3d_kitti", "unet3d_nyu", "unet2d", "OccDepth", "efficientnet",
             "flosp_depth", "flosp_depth.flosp_depth"]
    models = importlib.import_module("occdepth_b200.models")
    root = sys.modules.get("occdepth")
    if root is None:
        try:
            spec = importlib.util.find_spec("occdepth")
        except (ImportError, ValueError):
            spec = None
        if spec is not None:
            root = importlib.import_module("occdepth")          # the reference tree (namespace or regular package)
        else:
            root = types.ModuleType("occdepth")
            root.__path__ = []                                  # a package: sub-imports raise ModuleNotFoundError
            sys.modules["occdepth"] = root
    if not hasattr(root, "__path__"):
        root.__path__ = []
    stale = [k for k in sys.modules if k == "occdepth.models" or k.startswith("occdepth.models.")]
    for k in stale:                                             # a reference copy imported earlier is replaced
        del sys.modules[k]
    sys.modules["occdepth.models"] = models
    root.models = models
    for n in names:
        try:
            m = importlib.import_module("occdepth_b200.models." + n)
        except ImportError:
            continue
        sys.modules["occdepth.models." + n] = m
    return models
