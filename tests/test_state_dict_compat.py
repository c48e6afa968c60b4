"""The drop-in boundary: every module of occdepth_b200.models must expose exactly the reference's state_dict keys,
shapes and dtypes, in order (released checkpoints are loaded with strict=True, scripts/eval.py:65-70).  The
reference's layout is stored in tests/golden/state_dict_layout.json (oracle/gen_golden.py, run where the original
project is importable)."""
import copy
import json
import os
import types

import pytest

from oracle import gen_golden

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LAYOUT = json.load(open(os.path.join(G, "state_dict_layout.json")))
CASES = dict(gen_golden.state_dict_cases())


def _product():
    import occdepth_b200.models.OccDepth as OccDepth
    import occdepth_b200.models.flosp_depth as flosp_pkg
    import occdepth_b200.models.flosp_depth.flosp_depth as flosp_depth
    import occdepth_b200.models.unet2d as unet2d
    import occdepth_b200.models.unet3d_kitti as unet3d_kitti
    import occdepth_b200.models.unet3d_nyu as unet3d_nyu
    return types.SimpleNamespace(OccDepth=OccDepth, flosp_depth=flosp_depth, unet2d=unet2d, unet3d_kitti=unet3d_kitti,
                                 unet3d_nyu=unet3d_nyu, flosp_conf=flosp_pkg.flosp_depth_conf_map)


def _same(name):
    import occdepth_b200.models.flosp_depth.flosp_depth as mfd
    saved = copy.deepcopy(mfd.flosp_depth_conf_map)
    try:
        m = CASES[name](_product())
    finally:       # OccDepth mutates the module-level conf dicts in place (as the reference does)
        for k in mfd.flosp_depth_conf_map:
            mfd.flosp_depth_conf_map[k].clear()
            mfd.flosp_depth_conf_map[k].update(saved[k])
    got = gen_golden.state_dict_layout(m)    # (entries, digest of the ordered keys / shapes / dtypes)
    assert got == LAYOUT["modules"][name]
    return got[0]


def test_unet3d_keys():
    assert _same("unet3d_kitti") > 500
    assert _same("unet3d_nyu") > 500
    assert _same("unet3d_kitti_ps1") > 300      # project_scale 1 -> Convblock3d


@pytest.mark.parametrize("backbone", ["tf_efficientnet_b3_ns", "tf_efficientnet_b4_ns", "tf_efficientnet_b5_ns",
                                      "tf_efficientnet_b7_ns"])
def test_unet2d_keys(backbone):
    assert _same("unet2d_" + backbone) > 600


def test_flosp_depth_keys():
    from occdepth_b200.models.flosp_depth import flosp_depth_conf_map
    for ds in ("kitti", "NYU"):
        assert json.loads(json.dumps(flosp_depth_conf_map[ds])) == LAYOUT["conf_map"][ds]
        assert _same("flosp_depth_" + ds) == 56


@pytest.mark.parametrize("variant", ["kitti_flosp", "kitti_flosp_depth", "nyu_flosp"])
def test_occdepth_keys(variant):
    assert _same("occdepth_" + variant) > 1800
