"""Class map written by the classifier's epilogue (OCCD_OUT1_CLASS_U16, OccDepth.predict_classes) against planar logits
+ occd_argmax_classes, bit for bit: per kernel family at the launch level (channel counts, batch, residual, both
schedules, ties, NaN, the label remap, the refusal), per shipped configuration at the model level, under the X-slab
partition, and through serving.FramePipeline."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

import gpu_cases as G
from occdepth_b200 import _lib
from occdepth_b200.engine import ClassMapUnsupported, ConvOp, Plan, conv_taps
from occdepth_b200.models.OccDepth import OccDepth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IMPLS = {"simt": _lib.CONV_IMPL_SIMT, "tc": _lib.CONV_IMPL_TC, "tcx": _lib.CONV_IMPL_TCX,
         "halo": _lib.CONV_IMPL_HALO, "halox": _lib.CONV_IMPL_HALOX}


def _u16_equal(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _pair(precision, impl, dims, Cin, w, bias, res1=False, lut=None):
    """(class map of the fused launch, class map of the planar launch + occd_argmax_classes, plan info)"""
    B, D, H, W = dims
    Cout = bias.numel()
    plan = Plan(torch.device("cuda"), precision=precision)
    x = plan.alloc(B, D, H, W, Cin)
    g = torch.Generator(device="cuda").manual_seed(1)
    x.buf.copy_(G.rnd(precision)(torch.randn(x.buf.shape, device="cuda", generator=g)))
    r = None
    if res1:
        r = plan.alloc(B, D, H, W, Cout)
        r.buf.copy_(G.rnd(precision)(torch.randn(r.buf.shape, device="cuda", generator=g)))
    taps, ws = conv_taps(w, (1, 1, 1), (1, 1, 1))
    logits = torch.empty(B, Cout, D, H, W, dtype=torch.float32, device="cuda")
    cls = torch.empty(B, D, H, W, dtype=torch.uint16, device="cuda")
    kw = dict(res1=r, impl=impl)
    op_p = ConvOp([x], taps, ws, bias, (D, H, W), out1=logits, out1_mode="planar", **kw)
    if op_p.info()["N_tile"] < op_p.desc.Cout_pad and impl == _lib.CONV_IMPL_TC:
        with pytest.raises(ClassMapUnsupported):       # the planner split the channels over N tiles
            ConvOp([x], taps, ws, bias, (D, H, W), out1=cls, out1_mode="classes", **kw)
        return None, None, op_p.info()
    op_c = ConvOp([x], taps, ws, bias, (D, H, W), out1=cls, out1_mode="classes", lut=lut, **kw)
    # same kernel, same tiles (the SIMT kernel has none: with a class map it runs one thread per position)
    assert op_c.impl == op_p.impl and (impl == _lib.CONV_IMPL_SIMT or op_c.info() == op_p.info())
    st = _lib.stream_ptr()
    op_p.run(st)
    op_c.run(st)
    want = OccDepth.class_map(logits, lut)
    torch.cuda.synchronize()
    return cls, want, op_c.info()


def _weights(Cout, Cin, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(Cout, Cin, 3, 3, 3, generator=g) * 0.2).cuda(), torch.randn(Cout, generator=g).cuda()


CASES = [(impl, Cout) for impl in ("simt", "tc", "halo", "halox") for Cout in (2, 12, 20, 13)] + \
        [("tcx", 20), ("tcx", 61)]


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("impl,Cout", CASES)
def test_kernel_class_map_equals_argmax_of_logits(impl, Cout, precision):
    Cin = 16
    w, b = _weights(Cout, Cin)
    for res1 in (False, True):
        got, want, _ = _pair(precision, IMPLS[impl], (2, 4, 6, 32), Cin, w, b, res1=res1)
        if got is None:         # refused, as it must be: the per-tap planner chose N tiles narrower than Cout_pad
            continue
        assert _u16_equal(got, want), (impl, Cout, res1, int((got.int() != want.int()).sum()))


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_per_tap_kernel_both_schedules_and_n_tiles(precision):
    """the per-tap kernel's cooperative and ping-pong schedules, N tiles 16 .. 256 (a class map needs Cout_pad == N)"""
    seen = set()
    for Cout, dims in ((12, (2, 4, 6, 32)), (20, (2, 4, 6, 32)), (20, (2, 16, 64, 64)), (100, (2, 16, 64, 64)),
                       (250, (1, 8, 16, 32))):
        w, b = _weights(Cout, 32, seed=Cout)
        got, want, info = _pair(precision, _lib.CONV_IMPL_TC, dims, 32, w, b, res1=True)
        if got is None:
            continue
        assert _u16_equal(got, want), (Cout, dims, info)
        seen.add(info["schedule"])
    assert seen == {"cooperative", "pingpong"}, seen


@pytest.mark.parametrize("impl", list(IMPLS))
def test_ties_nan_and_label_remap(impl):
    """zero weights + equal biases: exact ties resolve to the first index; a NaN logit behaves as in
    occd_argmax_classes (channel 0 wins, later NaNs are skipped); the remap is uint16(lut[class])"""
    Cout, Cin = 20, 16
    w = torch.zeros(Cout, Cin, 3, 3, 3, device="cuda")
    for bias, first in (([0.0, 1.0, 3.0, 3.0, 3.0] + [-1.0] * 15, 2), ([5.0] * 20, 0),
                        ([float("nan"), 1.0] + [7.0] * 18, 0), ([1.0, float("nan"), 2.0] + [2.0] * 17, 2)):
        b = torch.tensor(bias, device="cuda")
        got, want, _ = _pair("tf32", IMPLS[impl], (1, 4, 6, 32), Cin, w, b)
        if got is None:
            continue
        assert _u16_equal(got, want) and bool((got.int() == first).all()), (impl, bias)
    lut = list(np.random.default_rng(0).permutation(np.arange(100, 300))[:Cout])
    w, b = _weights(Cout, Cin)
    got, want, _ = _pair("bf16", IMPLS[impl], (2, 4, 6, 32), Cin, w, b, lut=lut)
    assert got is None or (_u16_equal(got, want) and int(got.int().min()) >= 100)


def test_refusal_and_fallback():
    """a class map the kernel cannot write (Cout beyond one N tile) is refused without a launch; Plan.conv then plans
    logits + occd_argmax_classes and returns the same map"""
    Cout, Cin = 300, 32
    w, b = _weights(Cout, Cin)
    plan = Plan(torch.device("cuda"), precision="tf32")
    x = plan.alloc(1, 4, 6, 32, Cin)
    x.buf.copy_(G.tf32r(torch.randn(x.buf.shape, device="cuda")))
    cls = torch.empty(1, 4, 6, 32, dtype=torch.uint16, device="cuda")
    taps, ws = conv_taps(w, (1, 1, 1), (1, 1, 1))
    with pytest.raises(ClassMapUnsupported):
        ConvOp([x], taps, ws, b, (4, 6, 32), out1=cls, out1_mode="classes", impl=_lib.CONV_IMPL_TC)
    plan.conv(x, w, b, padding=1, out1=cls, out1_mode="classes", no_out0=True, name="wide", impl=_lib.CONV_IMPL_TC)
    assert [op.name for op in plan.ops] == ["wide", "occd_argmax_classes"]
    logits = torch.empty(1, Cout, 4, 6, 32, device="cuda")
    ref = Plan(torch.device("cuda"), precision="tf32")
    ref.add(ConvOp([x], taps, ws, b, (4, 6, 32), out1=logits, out1_mode="planar", impl=_lib.CONV_IMPL_TC))
    plan.run()
    ref.run()
    assert _u16_equal(cls, OccDepth.class_map(logits))


# ---- model level -------------------------------------------------------------------------------------------------
NAMES = ["nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti", "kitti_b3_f24_flospdepth_mono_2080ti",
         "kitti_b7_f64_flosp_a100", "kitti_b7_f64_flospdepth_a100", "nyu_b7_f200_v100"]
_MODELS = {}


def _sc():
    p = os.path.join(ROOT, "tools")
    if p not in sys.path:
        sys.path.insert(0, p)
    import shipped_configs
    return shipped_configs


def _case(name, **kw):
    key = (name, tuple(sorted(kw.items())))
    if key not in _MODELS:
        _MODELS.clear()
        gc.collect()
        torch.cuda.empty_cache()
        sc = _sc()
        m, batch, _ = sc.make_case(name, **kw)
        batch = sc.to_cuda(batch)
        if kw.get("infer_mode"):
            # what a deployment supplies instead of camera matrices: one sampling grid per camera and the scaled pixel
            # sizes
            X, Y, Z = (int(v) for v in m.flosp_depth.voxel_num.tolist())
            V = batch["img"].shape[1]
            g = torch.Generator().manual_seed(3)
            batch["grids"] = [(torch.rand(1, X, Y, Z, 3, generator=g) * 2.4 - 1.2).cuda() for _ in range(V)]
            batch["scaled_pixel_size"] = (torch.rand(V, 1, generator=g) + 0.5).cuda()
        _MODELS[key] = (m.cuda(), batch)
    return _MODELS[key]


def _count_builds(m, monkeypatch):
    n = [0]
    orig = m._build

    def counted(*a, **k):
        n[0] += 1
        return orig(*a, **k)
    monkeypatch.setattr(m, "_build", counted)
    return n


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("name", NAMES)
def test_predict_classes_shipped(name, precision, monkeypatch):
    m, batch = _case(name)
    m.set_precision(precision)
    builds = _count_builds(m, monkeypatch)
    with torch.no_grad():
        want = m.class_map(m(batch)["ssc_logit"])
        got = m.predict_classes(batch)
        assert _u16_equal(got, want), int((got.int() != want.int()).sum())
        # alternating forward and predict_classes replays both plans
        for _ in range(2):
            assert _u16_equal(m.class_map(m(batch)["ssc_logit"]), want)
            assert _u16_equal(m.predict_classes(batch), want)
    assert builds[0] == 2
    (plan, *_), = m._class_plans().values()
    names = [getattr(op, "name", "") for op in plan.ops]
    assert "occd_argmax_classes" not in names and not any("to_planar" in n for n in names)
    assert plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16
    inv = np.random.default_rng(1).permutation(256)[:m.n_classes]
    with torch.no_grad():
        assert _u16_equal(m.predict_classes(batch, inv), m.class_map(m(batch)["ssc_logit"], inv))
    m.invalidate_plans()


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_predict_classes_infer_mode_and_occluded_head(precision):
    for name, kw in (("kitti_b3_f32_flospdepth_2080ti", dict(infer_mode=True, img_hw=(96, 320), full=(64, 64, 16))),
                     ("kitti_b3_f24_flospdepth_mono_2080ti", dict(img_hw=(96, 320), full=(64, 64, 16)))):
        m, batch = _case(name, **kw)
        if not kw.get("infer_mode"):
            # the occluded head (not in a shipped YAML): built with the same weights recipe
            m.net_3d_decoder.occluded_cls = True
            from occdepth_b200.models.modules import SegmentationHeadOccludedCLS
            f = m.feature
            m.net_3d_decoder.occluded_head = SegmentationHeadOccludedCLS(f // 2, f // 2, m.n_classes, [1, 2, 3]).cuda().eval()
        m.set_precision(precision)
        with torch.no_grad():
            res = m(batch)
            want = m.class_map(res["ssc_logit"])
            assert _u16_equal(m.predict_classes(batch), want), name
        if not kw.get("infer_mode"):
            assert "occluded_logit" in res
        _MODELS.clear()


def test_param_change_rebuilds_the_class_plan(monkeypatch):
    m, batch = _case("kitti_b3_f24_flospdepth_mono_2080ti", img_hw=(96, 320), full=(64, 64, 16))
    m.set_precision("bf16")
    with torch.no_grad():
        a = m.predict_classes(batch)
        builds = _count_builds(m, monkeypatch)
        m.predict_classes(batch)
        assert builds[0] == 0
        w = m.net_3d_decoder.ssc_head.conv_classes.bias
        w.copy_(w + 10.0 * torch.arange(w.numel(), device=w.device))
        b = m.predict_classes(batch)
        assert builds[0] == 1 and len(m._class_plans()) == 1
        assert _u16_equal(b, m.class_map(m(batch)["ssc_logit"])) and not _u16_equal(a, b)
    _MODELS.clear()


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_class_maps_concatenate_to_the_whole(monkeypatch, name, world, precision):
    from occdepth_b200.parallel import SimSlabGroup
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    m, batch = _case(name)
    m.set_precision(precision)
    with torch.no_grad():
        whole = m.predict_classes(batch)
    m.invalidate_plans()
    img = batch["img"]
    B, V, _, H, W = img.shape
    pp = batch["projected_pix_%d" % m.project_scale]
    fm = batch["fov_mask_%d" % m.project_scale]
    N, P = pp[0].shape[1], pp[0].shape[2]
    grp = SimSlabGroup(world, halo=3)
    ents = []
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                ents.append(m._build(B, V, H, W, N, P, img.device, batch, classes=("classes", None)))
    finally:
        m.__dict__.pop("slab_ctx", None)
    for e in ents:
        m._stage(e, batch, img, pp, fm, img.device)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    torch.cuda.synchronize()
    got = torch.cat([e[4] for e in ents], 1)
    del ents
    gc.collect()
    assert _u16_equal(got, whole)


def test_frame_pipeline_classes_kitti_flosp():
    """FramePipeline(classes=True): frame by frame what predict_classes returns for the same inputs (flosp model: the
    pipeline's inputs are the image, the indices and the FOV masks)"""
    from occdepth_b200.serving import FramePipeline
    m, batch = _case("kitti_b7_f64_flosp_a100", img_hw=(96, 320), full=(64, 64, 16))
    m.set_precision("bf16")
    inv = np.arange(20)[::-1].copy()
    g = torch.Generator().manual_seed(5)
    frames = []
    for _ in range(3):
        img = torch.randn(batch["img"].shape, generator=g)
        frames.append((img.pin_memory(), batch["projected_pix_2"][0].cpu().pin_memory(),
                       batch["fov_mask_2"][0].cpu().pin_memory()))
    pipe = FramePipeline(m, frames[0][0].shape, frames[0][1].shape, frames[0][2].shape, classes=True, inv_map=inv)
    got = {}
    for i, f in enumerate(frames):
        t = pipe.submit(*f)
        if t is not None:
            got[t] = pipe.result(t).clone()
    t = pipe.flush()
    got[t] = pipe.result(t).clone()
    assert sorted(got) == [0, 1, 2]
    for i, (img, pix, fov) in enumerate(frames):
        with torch.no_grad():
            want = m.predict_classes({"img": img.cuda(), "projected_pix_2": [pix.cuda()], "fov_mask_2": [fov.cuda()]},
                                     inv).cpu()
        assert got[i].dtype == torch.uint16 and _u16_equal(got[i], want), i
    _MODELS.clear()
