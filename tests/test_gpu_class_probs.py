"""Class probabilities (OCCD_OUT1_CLASS_U16_PROBS): every class's softmax probability, written by the classifier's
epilogue beside the class map.  Single launches: the mode-5 map is the mode-3 map bit for bit, on the same kernel, tile
and schedule, the probability at the map's class is the mode-4 launch's confidence bit for bit, and every probability
is within one float16 ulp of occd_class_probs over the planar logits of the same descriptor (bit for bit where the
epilogue takes the channels in one thread's ascending order; the two-thread merges sum s in another order).
Whole models: within one float16 ulp of softmax(ssc_logit) of the same plan, the probability at the map's class is
the confidence, and batches, pipelines and the X-slab partition give the bytes of the one-GPU predict_frame."""
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
from occdepth_b200.models.modules import split_probs
from occdepth_b200.parallel import SimSlabGroup

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402

IMPLS = {"simt": _lib.CONV_IMPL_SIMT, "tc": _lib.CONV_IMPL_TC, "tcx": _lib.CONV_IMPL_TCX,
         "halo": _lib.CONV_IMPL_HALO, "halox": _lib.CONV_IMPL_HALOX}
RELEASED = ["nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti"]


def _sc():
    import shipped_configs
    return shipped_configs


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _same(a, b):
    """bit-identical (uint16 maps or float16 probabilities; NaN payloads included)"""
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def check_probs(probs, logits):
    """probs float16 [B, C, ...] against logits fp32 [B, C, ...]: at most one float16 ulp from the float64 softmax,
    NaN where it is NaN; returns the largest absolute difference"""
    p = torch.softmax(logits.double(), dim=1)
    assert probs.dtype == torch.float16 and probs.shape == p.shape
    nan_p, nan_q = torch.isnan(p), torch.isnan(probs)
    assert torch.equal(nan_p, nan_q), int((nan_p != nan_q).sum())
    h = p[~nan_p].half().view(torch.int16).int()         # non-negative float16: bits step by one ulp
    q = probs[~nan_p].view(torch.int16).int()
    bad = (q - h).abs() > 1
    assert not bool(bad.any()), (int(bad.sum()), probs[~nan_p][bad][:5].tolist(), p[~nan_p][bad][:5].tolist())
    return float((probs[~nan_p].double() - p[~nan_p]).abs().max()) if bool((~nan_p).any()) else 0.0


def check_top_is_conf(cmap, probs, conf):
    """the probability at the map's class is the confidence, bit for bit (the map without a remap)"""
    top = probs.gather(1, cmap.long().unsqueeze(1)).squeeze(1)
    assert _same(top, conf)


# ---- single launches ---------------------------------------------------------------------------------------------
def _launches(precision, impl, dims, Cin, w, bias, dil=1, res1=False):
    """planar logits, the mode-3 map, the mode-4 confidence and the mode-5 (map, probs) of one descriptor, or None
    where the class map is refused"""
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
    taps, ws = conv_taps(w, (dil,) * 3, (dil,) * 3)
    logits = torch.empty(B, Cout, D, H, W, dtype=torch.float32, device="cuda")
    cls = torch.empty(B, D, H, W, dtype=torch.uint16, device="cuda")
    both = torch.full(((1 + Cout) * B, D, H, W), 0xFFFF, dtype=torch.uint16, device="cuda")
    kw = dict(res1=r, impl=impl)
    op_p = ConvOp([x], taps, ws, bias, (D, H, W), out1=logits, out1_mode="planar", **kw)
    try:
        op_c = ConvOp([x], taps, ws, bias, (D, H, W), out1=cls, out1_mode="classes", **kw)
    except ClassMapUnsupported:
        with pytest.raises(ClassMapUnsupported):
            ConvOp([x], taps, ws, bias, (D, H, W), out1=both, out1_mode="classes_probs", **kw)
        return None
    op_k = ConvOp([x], taps, ws, bias, (D, H, W), out1=both, out1_mode="classes_probs", **kw)
    conf = torch.empty(2, B, D, H, W, dtype=torch.uint16, device="cuda")
    op_f = ConvOp([x], taps, ws, bias, (D, H, W), out1=conf, out1_mode="classes_conf", **kw)
    assert op_k.impl == op_c.impl == op_p.impl == op_f.impl
    assert impl == _lib.CONV_IMPL_SIMT or op_k.info() == op_c.info() == op_p.info() == op_f.info()
    st = _lib.stream_ptr()
    for op in (op_p, op_c, op_k, op_f):
        op.run(st)
    torch.cuda.synchronize()
    cmap, probs = split_probs(both, B)
    return logits, cls, cmap, probs, conf[1].view(torch.float16), op_k.info()


def _weights(Cout, Cin, seed=0, scale=0.2):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(Cout, Cin, 3, 3, 3, generator=g) * scale).cuda(), torch.randn(Cout, generator=g).cuda()


def _check_launch(res):
    logits, cls, cmap, probs, conf, info = res
    assert _same(cmap, cls), (info, int((cmap.int() != cls.int()).sum()))
    rmap, rprobs = OccDepth.class_map(logits, probabilities=True)
    assert _same(rmap, cls)
    nan = torch.isnan(rprobs)
    assert torch.equal(torch.isnan(probs), nan)
    ulps = (probs[~nan].view(torch.int16).int() - rprobs[~nan].view(torch.int16).int()).abs()
    assert ulps.numel() == 0 or int(ulps.max()) <= 1, (info, int((ulps > 1).sum()))
    check_probs(probs, logits)
    check_top_is_conf(cmap, probs, conf)
    return info


KCASES = [(impl, Cout) for impl in ("simt", "tc", "halo", "halox") for Cout in (20, 12, 13)] + \
         [("tcx", 20), ("tcx", 61)]


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("impl,Cout", KCASES)
def test_kernel_probs(impl, Cout, precision):
    w, b = _weights(Cout, 16)
    for res1 in (False, True):
        res = _launches(precision, IMPLS[impl], (2, 4, 6, 32), 16, w, b, res1=res1)
        if res is not None:
            _check_launch(res)


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_per_tap_kernel_both_schedules(precision):
    seen = set()
    for Cout, dims in ((12, (2, 4, 6, 32)), (20, (2, 4, 6, 32)), (20, (2, 16, 64, 64)), (13, (2, 16, 64, 64))):
        w, b = _weights(Cout, 32, seed=Cout)
        res = _launches(precision, _lib.CONV_IMPL_TC, dims, 32, w, b, res1=True)
        if res is not None:
            seen.add(_check_launch(res)["schedule"])
    assert seen == {"cooperative", "pingpong"}, seen


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("impl", ["halox", "tcx"])
@pytest.mark.parametrize("d", (1, 2, 3))
def test_xpacked_dilations(d, impl, precision):
    seen = set()
    for dims in ((2, 8, 16), (40, 256, 16), (2, 8, 32), (40, 256, 32)):
        w, b = _weights(20, 32, seed=d, scale=0.05)
        try:
            res = _launches(precision, IMPLS[impl], (1,) + dims, 32, w, b, dil=d)
        except RuntimeError as e:          # the planar plan itself is refused (a shape this kernel does not take)
            assert impl == "tcx", e
            continue
        if res is not None:
            seen.add(_check_launch(res)["schedule"])
    if impl == "halox":
        assert seen == {"cooperative", "pingpong"}, seen


def test_ties_nan_inf_and_remap():
    """zero weights and chosen biases: ties, NaN, +inf and -inf; the remap relabels the map only"""
    Cout, Cin = 20, 16
    w = torch.zeros(Cout, Cin, 3, 3, 3, device="cuda")
    nan, inf = float("nan"), float("inf")
    for bias in ([0.0, 1.0, 3.0, 3.0, 3.0] + [-1.0] * 15, [5.0] * 20, [nan, 1.0] + [7.0] * 18,
                 [1.0, nan, 2.0] + [2.0] * 17, [1.0, inf] + [0.0] * 18, [-inf] * 19 + [2.0], [-inf] * 20,
                 [1e30, -1e30] + [0.0] * 18, [-60.0] * 10 + [40.0] * 10):
        b = torch.tensor(bias, device="cuda")
        for impl in IMPLS:
            res = _launches("tf32", IMPLS[impl], (1, 4, 6, 32), Cin, w, b)
            if res is not None:
                _check_launch(res)
    wr, br = _weights(Cout, Cin)
    logits = _launches("tf32", _lib.CONV_IMPL_SIMT, (2, 4, 6, 32), Cin, wr, br)[0]
    inv = np.random.default_rng(0).permutation(256)[:Cout]
    m0, p0 = OccDepth.class_map(logits, probabilities=True)
    m1, p1 = OccDepth.class_map(logits, inv, probabilities=True)
    assert _same(p0, p1) and _same(m1, OccDepth.class_map(logits, inv)) and _same(m0, OccDepth.class_map(logits))


def test_fallback_probs():
    """a class map beyond one N tile: logits + occd_class_probs give the same bytes as class_map"""
    Cout, Cin = 300, 32
    w, b = _weights(Cout, Cin)
    plan = Plan(torch.device("cuda"), precision="tf32")
    x = plan.alloc(1, 4, 6, 32, Cin)
    x.buf.copy_(G.tf32r(torch.randn(x.buf.shape, device="cuda")))
    both = torch.empty((1 + Cout) * 1, 4, 6, 32, dtype=torch.uint16, device="cuda")
    plan.conv(x, w, b, padding=1, out1=both, out1_mode="classes_probs", no_out0=True, name="wide",
              impl=_lib.CONV_IMPL_TC)
    assert [op.name for op in plan.ops] == ["wide", "occd_class_probs"]
    logits = torch.empty(1, Cout, 4, 6, 32, device="cuda")
    taps, ws = conv_taps(w, (1, 1, 1), (1, 1, 1))
    ref = Plan(torch.device("cuda"), precision="tf32")
    ref.add(ConvOp([x], taps, ws, b, (4, 6, 32), out1=logits, out1_mode="planar", impl=_lib.CONV_IMPL_TC))
    plan.run()
    ref.run()
    m, p = OccDepth.class_map(logits, probabilities=True)
    cmap, probs = split_probs(both, 1)
    assert _same(cmap, m) and _same(probs, p)


# ---- whole models --------------------------------------------------------------------------------------------------
MODEL_CASES = [(n, p) for n in _sc().CONFIGS for p in G.PRECISIONS]


@pytest.mark.parametrize("name,precision", MODEL_CASES)
def test_predict_classes_probs_shipped(name, precision):
    sc = _sc()
    _free()
    m, batch, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    batch = sc.to_cuda(batch)
    inv = np.random.default_rng(1).permutation(256)[:m.n_classes]
    with torch.no_grad():
        logits = m(batch)["ssc_logit"]
        plain = m.predict_classes(batch)
        cmap, probs = m.predict_classes(batch, probabilities=True)
        assert _same(cmap, plain), int((cmap.int() != plain.int()).sum())
        assert probs.shape == logits.shape
        diff = check_probs(probs, logits)
        print("%s %s: max |probs - softmax(ssc_logit)| = %.3g" % (name, precision, diff))
        check_top_is_conf(cmap, probs, m.predict_classes(batch, confidence=True)[1])
        cmap_i, probs_i = m.predict_classes(batch, inv, probabilities=True)
        want_i = torch.as_tensor(inv.astype(np.int64), device="cuda")[plain.long()].to(torch.uint16)
        assert _same(probs_i, probs) and _same(cmap_i, want_i)
    (plan, *_), = m._class_plans().values()
    assert plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16_PROBS or plan.ops[-1].name == "occd_class_probs"
    del m, batch, logits
    _free()


# ---- camera frames -------------------------------------------------------------------------------------------------
def _camera_frames(sc, spec):
    if spec["dataset"] == "NYU":
        frames = [nyu_frame(1), nyu_frame(2), nyu_frame(3)]
        frames[1]["cam_pose"][0, 3] += 0.2
        return [dict(f, img_hw=sc.NYU_IMG) for f in frames]
    H, W = sc.KITTI_IMG
    geo = kitti_geometry(H, W, sc.KITTI_FULL)
    frames = [kitti_frame(spec["views"], H, W, 1), kitti_frame(spec["views"], H, W, 2),
              kitti_frame(spec["views"], H, W, 3, shift=0.3)]
    return [dict(f, **geo) for f in frames]


def _drain(pipe, items):
    got = {}
    for it in items:
        t = pipe.submit(it)
        if t is not None:
            got[t] = tuple(x.clone() for x in pipe.result(t))
    t = pipe.flush()
    got[t] = tuple(x.clone() for x in pipe.result(t))
    return got


@pytest.mark.parametrize("name", RELEASED)
def test_camera_frames_probs(name):
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    _free()
    spec = sc.CONFIGS[name]
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, spec)
    with torch.no_grad():
        want = [m.predict_frame(f, probabilities=True) for f in frames]
        for f, (cmap, probs) in zip(frames, want):
            assert _same(cmap, m.predict_frame(f))
            check_probs(probs, m.predict_frame(f, classes=False)["ssc_logit"])
        for B in (2, 3):
            cmaps, probs = m.predict_frames(frames[:B], probabilities=True)
            for i in range(B):
                assert _same(cmaps[i:i + 1], want[i][0]) and _same(probs[i:i + 1], want[i][1]), (B, i)
    with pytest.raises(ValueError, match="no probability columns"):
        CameraPipeline(m, img_hw=frames[0]["img_hw"], output="voxels", probabilities=True)
    with pytest.raises(ValueError, match="already hold the confidence"):
        CameraPipeline(m, img_hw=frames[0]["img_hw"], confidence=True, probabilities=True)
    pipe = CameraPipeline(m, img_hw=frames[0]["img_hw"], probabilities=True)
    got = _drain(pipe, frames)
    assert sorted(got) == [0, 1, 2]
    for i, (cmap, probs) in enumerate(want):
        assert got[i][1].dtype == torch.float16
        assert _same(got[i][0], cmap.cpu()) and _same(got[i][1], probs.cpu()), i
    del pipe
    pipe = CameraPipeline(m, img_hw=frames[0]["img_hw"], probabilities=True, batch=2)
    got = _drain(pipe, [frames[:2], frames[2:]])        # a full list, then a short one
    assert got[1][0].shape[0] == 1
    cm = torch.cat([got[0][0], got[1][0]])
    pr = torch.cat([got[0][1], got[1][1]])
    for i, (cmap, probs) in enumerate(want):
        assert _same(cm[i:i + 1], cmap.cpu()) and _same(pr[i:i + 1], probs.cpu()), i
    del m, pipe
    _free()


# ---- X-slab partition ----------------------------------------------------------------------------------------------
def _rank_entries(m, world, f, classes):
    grp = SimSlabGroup(world, halo=3)
    dev = f["imgs"].device
    ents = []
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad(), torch.cuda.device(dev):
                ents.append(m._build(1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["batch"], classes=classes))
    finally:
        m.__dict__.pop("slab_ctx", None)
    return ents


@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("kitti_b3_f32_flospdepth_2080ti", 3),
                                        ("nyu_b4_f100_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_probs(monkeypatch, name, world):
    """slab_output="slab": each rank's [1, C, X_slab, Y, Z], concatenated along X, is the one-GPU result"""
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, sc.CONFIGS[name])[:2]
    with torch.no_grad():
        want = [m.predict_frame(f, probabilities=True) for f in frames]
    m.invalidate_plans()
    dev = next(m.parameters()).device
    fs = [m._frame_inputs(f, dev) for f in frames]
    ents = _rank_entries(m, world, fs[0], m._class_key(None, probabilities=True))
    for f, (wmap, wprobs) in zip(fs, want):
        for e in ents:
            m._stage_frame(e, f)
        with torch.no_grad():
            SimSlabGroup.run_lockstep([e[0] for e in ents])
        torch.cuda.synchronize()
        parts = [split_probs(e[4], 1) for e in ents]
        assert _same(torch.cat([p[0] for p in parts], 1), wmap)
        assert _same(torch.cat([p[1] for p in parts], 2), wprobs)
    del ents, m
    _free()


@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("kitti_b3_f32_flospdepth_2080ti", 3),
                                        ("nyu_b4_f100_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_root_probs(monkeypatch, name, world):
    """slab_output="root": rank 0's whole (map, probs) is the one-GPU result, from one gather of 1 + C items"""
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, sc.CONFIGS[name])[:2]
    with torch.no_grad():
        want = [m.predict_frame(f, probabilities=True) for f in frames]
    m.invalidate_plans()
    dev = next(m.parameters()).device
    fs = [m._frame_inputs(f, dev) for f in frames]
    ents = _rank_entries(m, world, fs[0], m._class_key(None, root=True, probabilities=True))
    assert [op.name for op in ents[0][0].ops].count("gather_root") == 1
    for f, (wmap, wprobs) in zip(fs, want):
        for e in ents:
            m._stage_frame(e, f)
        with torch.no_grad():
            SimSlabGroup.run_lockstep([e[0] for e in ents])
        torch.cuda.synchronize()
        cmap, probs = split_probs(ents[0][4], 1)
        assert _same(cmap, wmap) and _same(probs, wprobs)
        assert all(e[4] is None for e in ents[1:])
    del ents, m
    _free()


# ---- model files ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,precision", [(n, p) for n in RELEASED for p in ("tf32", "bf16")])
def test_model_file_probs(name, precision, tmp_path):
    from occdepth_b200 import deploy
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    frames = _camera_frames(sc, sc.CONFIGS[name])
    with torch.no_grad():
        want = [m.predict_frame(f, probabilities=True) for f in frames]
        deploy.export(m, tmp_path / "probs.occd", frames[0], probabilities=True)
        deploy.export(m, tmp_path / "batch.occd", frames[:2], probabilities=True)
        deploy.export(m, tmp_path / "plain.occd", frames[0])
        with pytest.raises(ValueError, match="already hold the confidence"):
            deploy.export(m, tmp_path / "x.occd", frames[0], confidence=True, probabilities=True)
    pm = deploy.LoadedModel(tmp_path / "probs.occd")
    for i, (f, (wmap, wprobs)) in enumerate(zip(frames, want)):
        cmap, probs = pm.run_frames([f], probs=True)
        torch.cuda.synchronize()
        assert _same(cmap, wmap) and _same(probs, wprobs), i
        assert _same(pm.run_frames([f]), wmap)                # the map-only call on a probabilities file
    pm.close()
    bm = deploy.LoadedModel(tmp_path / "batch.occd")
    for fs, ws in ((frames[:2], want[:2]), (frames[2:], want[2:])):   # a full group, then a short one
        cmap, probs = bm.run_frames(fs, probs=True)
        torch.cuda.synchronize()
        for i, (wmap, wprobs) in enumerate(ws):
            assert _same(cmap[i:i + 1], wmap) and _same(probs[i:i + 1], wprobs), i
    bm.close()
    plain = deploy.LoadedModel(tmp_path / "plain.occd")
    with pytest.raises(RuntimeError, match="without probabilities"):
        plain.run_frames([frames[0]], probs=True)
    plain.close()
    del m
    _free()


@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_model_files_probs(name, world, tmp_path):
    """every rank's file, exported with probabilities, run in lock step on a local group: rank 0's whole (map,
    probs) is predict_frame's"""
    from occdepth_b200 import deploy
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, sc.CONFIGS[name])
    with torch.no_grad():
        want = [m.predict_frame(f, probabilities=True) for f in frames]
    paths = [tmp_path / ("r%d.occd" % r) for r in range(world)]
    grp = SimSlabGroup(world, halo=3)
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                deploy.export(m, paths[r], frames[0], slab_output="root", probabilities=True)
    finally:
        m.__dict__.pop("slab_ctx", None)
    comms = deploy.Comm.local(world)
    models = [deploy.LoadedModel(p, c) for p, c in zip(paths, comms)]
    for graph in (True, False):
        for i, (f, (wmap, wprobs)) in enumerate(zip(frames, want)):
            cmap, probs = deploy.run_frame_group(models, f, graph=graph, probs=True)
            torch.cuda.synchronize()
            assert _same(cmap, wmap) and _same(probs, wprobs), (graph, i)
    for x in models:
        x.close()
    del m
    _free()


# ---- pipelines -------------------------------------------------------------------------------------------------------
def test_frame_pipeline_probs():
    """FramePipeline takes the image, the indices and the FOV masks only: the configuration that needs nothing else"""
    from occdepth_b200.serving import FramePipeline
    name = "kitti_b7_f64_flosp_a100"
    sc = _sc()
    _free()
    m, batch, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    batch = sc.to_cuda(batch)
    ps = "%d" % m.project_scale
    img = batch["img"].cpu().pin_memory()
    pix = batch["projected_pix_" + ps][0].cpu().pin_memory()
    fov = batch["fov_mask_" + ps][0].cpu().pin_memory()
    with torch.no_grad():
        wmap, wprobs = m.predict_classes(batch, probabilities=True)
    with pytest.raises(ValueError, match=r"probabilities \(classes=True\)"):
        FramePipeline(m, img.shape, pix.shape, fov.shape, probabilities=True)
    pipe = FramePipeline(m, img.shape, pix.shape, fov.shape, classes=True, probabilities=True)
    got = {}
    for _ in range(3):
        t = pipe.submit(img, pix, fov)
        if t is not None:
            got[t] = tuple(x.clone() for x in pipe.result(t))
    t = pipe.flush()
    got[t] = tuple(x.clone() for x in pipe.result(t))
    assert sorted(got) == [0, 1, 2]
    for i in range(3):
        assert _same(got[i][0], wmap.cpu()) and _same(got[i][1], wprobs.cpu()), i
    del m, pipe
    _free()
