"""tests/conv_menu.py without a GPU: the menu it parses from csrc/conv_kernels.cuh is the one the N-tile test lists,
its cells are the compiled instantiations, and every case of the menu sweep plans on the SIMT kernel (the only one
that plans without a driver) and is evaluated by the float64 reference."""
import pytest
import torch

import conv_menu as M
import conv_replay as R
import test_gpu_conv_ntiles as NT


def test_parsed_menu_is_the_ntile_menu():
    menu, pp_max = M.parse_menu()
    assert menu == NT.MENU
    assert pp_max == 128
    cells = M.compiled_cells()
    per_precision = sum(len(t) for t in menu.values()) + sum(
        len([n for n in t if n <= pp_max]) for k, t in menu.items() if k != "halo") + 1
    assert len(cells) == 2 * per_precision == 86


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("family", M.FAMILIES)
def test_every_case_plans_on_simt(family, precision, monkeypatch):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    items = M.build(family, precision, torch.device("cpu"), simt=True)
    assert items
    for op, expect in items:
        assert op.impl == M.IMPL["simt"] and expect == {}
        sig = R.signature(op)
        D = dict(sig)
        assert D["kernel"] is None
        if D["B"] * D["Of"][0] * D["Of"][1] * D["Of"][2] * D["Cout"] <= 60000:
            R.fill(op, R.seed_of(sig))
            ref = R.reference(R.Snapshot(op))
            assert bool(ref.mask.any()) and bool(torch.isfinite(ref.v).all())

