"""Class-map output of the convolution epilogue (OCCD_OUT1_CLASS_U16) on the host: argument validation and the
refusals of occd_conv_plan_create, the label remap entry point, and the engine's choice between the fused map and the
logits + occd_argmax_classes fallback.  None of it needs a GPU: SIMT plans are built without a driver, and the
tensor-core plans answer before their tensor-map encode."""
import contextlib
import ctypes as C
import io

import pytest
import torch
import torch.nn as nn

from occdepth_b200 import _build, _lib

FAKE = 0x100000        # an aligned device address: plan creation never dereferences it


def _desc(impl, Cout=20, out1_mode=_lib.OUT1_CLASS_U16, out1=FAKE):
    d = _lib.ConvDesc()
    d.impl, d.dtype, d.n_src = impl, _lib.DTYPE_F32, 1
    d.src[0], d.src_C[0], d.src_cstride[0] = FAKE, 16, 16
    d.B, d.ID, d.IH, d.IW = 2, 4, 6, 32
    d.stride[:] = [1, 1, 1]
    d.omul[:] = [1, 1, 1]
    taps = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]
    d.n_taps = len(taps)
    for i, (a, b, c) in enumerate(taps):
        d.taps[i].src, d.taps[i].dz, d.taps[i].dy, d.taps[i].dx = 0, a, b, c
    d.weight, d.bias = FAKE, FAKE
    d.Cout, d.Cout_pad, d.Kpad = Cout, (Cout + 15) // 16 * 16, 16
    d.OD, d.OH, d.OW = 4, 6, 32
    d.ODf, d.OHf, d.OWf = 4, 6, 32
    d.out1_mode, d.out1, d.out1_C = out1_mode, out1, Cout
    return d


def _create(d):
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.occd_conv_plan_create(C.byref(d), C.byref(h))
    return rc, h, L.occd_last_error().decode()


def test_plan_create_validates_the_class_map_without_gpu():
    _build.build()
    L = _lib.lib()
    rc, h, msg = _create(_desc(_lib.CONV_IMPL_SIMT))
    assert rc == 0, msg
    try:
        lut = (C.c_int * 20)(*range(100, 120))
        assert L.occd_conv_plan_set_class_lut(h, lut, 20) == 0
        assert L.occd_conv_plan_set_class_lut(h, None, 0) == 0                 # back to plain class indices
        assert L.occd_conv_plan_set_class_lut(h, lut, 19) == _lib.ERR_ARG       # one label per class
    finally:
        L.occd_conv_plan_destroy(h)
    assert L.occd_conv_plan_set_class_lut(None, None, 0) == _lib.ERR_ARG
    rc, h, msg = _create(_desc(_lib.CONV_IMPL_SIMT, Cout=80))
    assert rc == 0, msg
    try:
        big = (C.c_int * 80)(*range(80))
        assert L.occd_conv_plan_set_class_lut(h, big, 80) == _lib.ERR_ARG       # a remap covers at most 64 classes
    finally:
        L.occd_conv_plan_destroy(h)
    rc, h, msg = _create(_desc(_lib.CONV_IMPL_SIMT, out1_mode=_lib.OUT1_F32_PLANAR))
    assert rc == 0, msg
    try:
        assert L.occd_conv_plan_set_class_lut(h, None, 0) == _lib.ERR_ARG       # no class map in this plan
    finally:
        L.occd_conv_plan_destroy(h)
    # bad arguments
    assert _create(_desc(_lib.CONV_IMPL_SIMT, out1=None))[0] == _lib.ERR_ARG
    assert _create(_desc(_lib.CONV_IMPL_SIMT, out1=FAKE + 1))[0] == _lib.ERR_ARG  # uint16 alignment
    assert _create(_desc(_lib.CONV_IMPL_SIMT, Cout=65536))[0] == _lib.ERR_ARG
    # what a kernel cannot do
    d = _desc(_lib.CONV_IMPL_SIMT)
    d.out0, d.out0_cstride = FAKE, 32
    rc, _, msg = _create(d)
    assert rc == _lib.ERR_UNSUPPORTED and "only output" in msg
    rc, _, msg = _create(_desc(_lib.CONV_IMPL_TC, Cout=300))                     # N tiles of 16 over 304 channels
    assert rc == _lib.ERR_UNSUPPORTED and "one N tile" in msg
    d = _desc(_lib.CONV_IMPL_TC)
    d.n_groups, d.group_tap0[0], d.group_tap0[1], d.group_tap0[2] = 2, 0, 9, 27
    d.omul[:] = [2, 2, 2]
    d.ODf, d.OHf, d.OWf = 8, 12, 64
    d.group_oadd[1][:] = [1, 1, 1]
    assert _create(d)[0] == _lib.ERR_UNSUPPORTED                                 # tap groups
    # the planar mode of the same descriptors is untouched: it reaches the tensor-map encode (no driver here)
    rc, _, msg = _create(_desc(_lib.CONV_IMPL_TC, Cout=300, out1_mode=_lib.OUT1_F32_PLANAR, out1=FAKE))
    assert rc != _lib.ERR_UNSUPPORTED, msg


def test_engine_fuses_the_class_map_or_falls_back(monkeypatch):
    """Plan.conv(out1_mode="classes"): one conv launch where the kernel writes the map; where plan creation refuses
    it, the plan writes logits into a buffer of its own and adds occd_argmax_classes"""
    from occdepth_b200.engine import ClassMapUnsupported, ConvOp, Plan
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    out = torch.empty(2, 4, 6, 32, dtype=torch.uint16)
    plan.conv(x, torch.randn(20, 16, 3, 3, 3), torch.randn(20), padding=1, out1=out, out1_mode="classes",
              lut=list(range(20)), no_out0=True, name="cls")
    assert [op.name for op in plan.ops] == ["cls"] and plan.ops[0].desc.out1_mode == _lib.OUT1_CLASS_U16

    taps = [(0, 0, 0, 0)]
    with pytest.raises(ClassMapUnsupported, match="one N tile"):
        ConvOp([x], taps, [torch.randn(300, 16)], torch.randn(300), (4, 6, 32), out1=out, out1_mode="classes",
               impl=_lib.CONV_IMPL_TC, name="wide")
    # the fallback: the refused launch is planned again with planar logits (the tensor-map encode of that plan is the
    # first step that needs a driver)
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "tc")
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    with pytest.raises(RuntimeError, match="cuTensorMapEncodeTiled unavailable") as ei:
        plan.conv(x, torch.randn(300, 16, 1, 1, 1), torch.randn(300), out1=out, out1_mode="classes", no_out0=True,
                  name="wide")
    assert not isinstance(ei.value, ClassMapUnsupported)


@pytest.mark.parametrize("cascade", [False, True])
def test_decoder_class_map_plan(monkeypatch, cascade):
    """the KITTI decoder in class-map mode ends in the fused classifier: no planar logits, no arg-max launch, no
    occluded head"""
    from occdepth_b200.engine import Plan
    from occdepth_b200.models.unet3d_kitti import UNet3D
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    with contextlib.redirect_stdout(io.StringIO()):
        m = UNet3D(20, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=False, cascade_cls=cascade,
                   occluded_cls=True).eval()
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(1, 16, 16, 8, 16)
    with torch.no_grad():
        y = m.emit(plan, x, classes=True, lut=list(range(20)))
    assert y.dtype == torch.uint16 and tuple(y.shape) == (1, 32, 32, 16)
    names = [getattr(op, "name", "") for op in plan.ops]
    last = "head.conv_classes.b" if cascade else "head.conv_classes"
    assert names[-1] == last and plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16
    assert "occd_argmax_classes" not in names and not any(n.startswith("occl.") for n in names)
