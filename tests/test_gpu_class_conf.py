"""Class-map confidence (OCCD_OUT1_CLASS_U16_CONF): each voxel's top-class softmax probability, written by the
classifier's epilogue beside the class map.  Against the planar logits of the same descriptor (single launches) or
forward()["ssc_logit"] (whole models): the map is bit for bit the mode-3 map, and the float16 confidence is float16(p)
or one of its float16 neighbours, p the float64 softmax maximum, NaN exactly where p is NaN.  Camera frames, the
X-slab partition and model files give the same bytes as the one-GPU predict_frame."""
import ctypes as C
import gc
import os
import struct
import sys

import numpy as np
import pytest
import torch

import gpu_cases as G
from occdepth_b200 import _lib, deploy
from occdepth_b200.engine import ClassMapUnsupported, ConvOp, Plan, conv_taps
from occdepth_b200.models.OccDepth import OccDepth
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
    """bit-identical (uint16 maps or float16 confidences; NaN payloads included)"""
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def check_conf(conf, logits):
    """conf float16 [B, ...] against logits fp32 [B, C, ...]: float16(p) or a float16 neighbour, NaN where p is NaN"""
    p = torch.softmax(logits.double(), dim=1).amax(dim=1)
    assert conf.dtype == torch.float16 and conf.shape == p.shape
    nan_p, nan_c = torch.isnan(p), torch.isnan(conf)
    assert torch.equal(nan_p, nan_c), int((nan_p != nan_c).sum())
    h = p[~nan_p].half().view(torch.int16).int()         # p is in [1/64, 1]: positive normals, bits step by one
    c = conf[~nan_p].view(torch.int16).int()
    bad = (c - h).abs() > 1
    assert not bool(bad.any()), (int(bad.sum()), conf[~nan_p][bad][:5].tolist(), p[~nan_p][bad][:5].tolist())


# ---- single launches ---------------------------------------------------------------------------------------------
def _launches(precision, impl, dims, Cin, w, bias, dil=1, res1=False):
    """planar logits, the mode-3 map and the mode-4 (map, conf) of one descriptor, or None where the class map is
    refused (the per-tap planner split the channels over N tiles)"""
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
    both = torch.empty(2, B, D, H, W, dtype=torch.uint16, device="cuda")
    kw = dict(res1=r, impl=impl)
    op_p = ConvOp([x], taps, ws, bias, (D, H, W), out1=logits, out1_mode="planar", **kw)
    try:
        op_c = ConvOp([x], taps, ws, bias, (D, H, W), out1=cls, out1_mode="classes", **kw)
    except ClassMapUnsupported:
        with pytest.raises(ClassMapUnsupported):
            ConvOp([x], taps, ws, bias, (D, H, W), out1=both, out1_mode="classes_conf", **kw)
        return None
    op_k = ConvOp([x], taps, ws, bias, (D, H, W), out1=both, out1_mode="classes_conf", **kw)
    assert op_k.impl == op_c.impl == op_p.impl
    assert impl == _lib.CONV_IMPL_SIMT or op_k.info() == op_c.info() == op_p.info()
    st = _lib.stream_ptr()
    for op in (op_p, op_c, op_k):
        op.run(st)
    torch.cuda.synchronize()
    return logits, cls, both[0], both[1].view(torch.float16), op_k.info()


def _weights(Cout, Cin, seed=0, scale=0.2):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(Cout, Cin, 3, 3, 3, generator=g) * scale).cuda(), torch.randn(Cout, generator=g).cuda()


def _check_launch(res):
    logits, cls, cmap, conf, info = res
    assert _same(cmap, cls), (info, int((cmap.int() != cls.int()).sum()))
    check_conf(conf, logits)
    return info


KCASES = [(impl, Cout) for impl in ("simt", "tc", "halo", "halox") for Cout in (20, 12, 13)] + \
         [("tcx", 20), ("tcx", 61)]


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("impl,Cout", KCASES)
def test_kernel_conf(impl, Cout, precision):
    Cin = 16
    w, b = _weights(Cout, Cin)
    for res1 in (False, True):
        res = _launches(precision, IMPLS[impl], (2, 4, 6, 32), Cin, w, b, res1=res1)
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
    """the x-packed epilogue's lane-pair merge at the dilations tests/test_gpu_xp_epilogue.py covers, both schedules"""
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
    """zero weights and chosen biases: ties, NaN in channel 0 and later, +inf and -inf; the remap leaves the
    confidence alone"""
    Cout, Cin = 20, 16
    w = torch.zeros(Cout, Cin, 3, 3, 3, device="cuda")
    nan, inf = float("nan"), float("inf")
    for bias in ([0.0, 1.0, 3.0, 3.0, 3.0] + [-1.0] * 15, [5.0] * 20, [nan, 1.0] + [7.0] * 18,
                 [1.0, nan, 2.0] + [2.0] * 17, [1.0, inf] + [0.0] * 18, [-inf] * 19 + [2.0], [-inf] * 20,
                 [1e30, -1e30] + [0.0] * 18):
        b = torch.tensor(bias, device="cuda")
        for impl in IMPLS:
            res = _launches("tf32", IMPLS[impl], (1, 4, 6, 32), Cin, w, b)
            if res is not None:
                _check_launch(res)
    # the remap: the conv plan's LUT and class_map's inv_map relabel the class only
    wr, br = _weights(Cout, Cin)
    logits = _launches("tf32", _lib.CONV_IMPL_SIMT, (2, 4, 6, 32), Cin, wr, br)[0]
    inv = np.random.default_rng(0).permutation(256)[:Cout]
    m0, c0 = OccDepth.class_map(logits, confidence=True)
    m1, c1 = OccDepth.class_map(logits, inv, confidence=True)
    assert _same(c0, c1) and _same(m1, OccDepth.class_map(logits, inv)) and _same(m0, OccDepth.class_map(logits))
    check_conf(c0, logits)


def test_fallback_conf():
    """a class map beyond one N tile: logits + occd_argmax_classes_conf give the same bytes as class_map"""
    Cout, Cin = 300, 32
    w, b = _weights(Cout, Cin)
    plan = Plan(torch.device("cuda"), precision="tf32")
    x = plan.alloc(1, 4, 6, 32, Cin)
    x.buf.copy_(G.tf32r(torch.randn(x.buf.shape, device="cuda")))
    both = torch.empty(2, 1, 4, 6, 32, dtype=torch.uint16, device="cuda")
    plan.conv(x, w, b, padding=1, out1=both, out1_mode="classes_conf", no_out0=True, name="wide",
              impl=_lib.CONV_IMPL_TC)
    assert [op.name for op in plan.ops] == ["wide", "occd_argmax_classes_conf"]
    logits = torch.empty(1, Cout, 4, 6, 32, device="cuda")
    taps, ws = conv_taps(w, (1, 1, 1), (1, 1, 1))
    ref = Plan(torch.device("cuda"), precision="tf32")
    ref.add(ConvOp([x], taps, ws, b, (4, 6, 32), out1=logits, out1_mode="planar", impl=_lib.CONV_IMPL_TC))
    plan.run()
    ref.run()
    m, c = OccDepth.class_map(logits, confidence=True)
    assert _same(both[0], m) and _same(both[1].view(torch.float16), c)


# ---- whole models --------------------------------------------------------------------------------------------------
MODEL_CASES = [(n, "tf32") for n in _sc().CONFIGS] + [(n, "bf16") for n in RELEASED]


@pytest.mark.parametrize("name,precision", MODEL_CASES)
def test_predict_classes_conf_shipped(name, precision):
    sc = _sc()
    _free()
    m, batch, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    batch = sc.to_cuda(batch)
    inv = np.random.default_rng(1).permutation(256)[:m.n_classes]
    with torch.no_grad():
        logits = m(batch)["ssc_logit"]
        plain = m.predict_classes(batch)
        cmap, conf = m.predict_classes(batch, confidence=True)
        assert _same(cmap, plain), int((cmap.int() != plain.int()).sum())
        assert _same(cmap, m.class_map(logits))
        check_conf(conf, logits)
        cmap_i, conf_i = m.predict_classes(batch, inv, confidence=True)
        want_i = torch.as_tensor(inv.astype(np.int64), device="cuda")[plain.long()].to(torch.uint16)
        assert _same(conf_i, conf) and _same(cmap_i, want_i)
        fmap, fconf = m.class_map(logits, confidence=True)
        assert _same(fmap, plain)
        check_conf(fconf, logits)
    (plan, *_), = m._class_plans().values()
    assert plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16_CONF
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


@pytest.mark.parametrize("name", RELEASED)
def test_camera_frames_conf(name):
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    _free()
    spec = sc.CONFIGS[name]
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, spec)
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=True) for f in frames]
        for f, (cmap, conf) in zip(frames, want):
            assert _same(cmap, m.predict_frame(f))
            check_conf(conf, m.predict_frame(f, classes=False)["ssc_logit"])
        with pytest.raises(ValueError):
            m.predict_frame(frames[0], classes=False, confidence=True)
    with pytest.raises(ValueError):
        CameraPipeline(m, img_hw=frames[0]["img_hw"], output="voxels", confidence=True)
    pipe = CameraPipeline(m, img_hw=frames[0]["img_hw"], confidence=True)
    got = {}
    for f in frames:
        t = pipe.submit(f)
        if t is not None:
            got[t] = tuple(x.clone() for x in pipe.result(t))
    t = pipe.flush()
    got[t] = tuple(x.clone() for x in pipe.result(t))
    assert sorted(got) == [0, 1, 2]
    for i, (cmap, conf) in enumerate(want):
        assert got[i][1].dtype == torch.float16
        assert _same(got[i][0], cmap.cpu()) and _same(got[i][1], conf.cpu()), i
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


def _run_ranks(m, ents, f):
    for e in ents:
        m._stage_frame(e, f)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    torch.cuda.synchronize()


@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("kitti_b3_f32_flospdepth_2080ti", 3),
                                        ("nyu_b4_f100_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_conf(monkeypatch, name, world):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    frames = _camera_frames(sc, sc.CONFIGS[name])[:2]
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=True) for f in frames]
    m.invalidate_plans()
    dev = next(m.parameters()).device
    fs = [m._frame_inputs(f, dev) for f in frames]
    ents = _rank_entries(m, world, fs[0], m._class_key(None, True))
    for f, (wmap, wconf) in zip(fs, want):
        _run_ranks(m, ents, f)
        got = torch.cat([e[4] for e in ents], 2)                 # [2, 1, X, Y, Z]
        assert _same(got[0], wmap) and _same(got[1].view(torch.float16), wconf)
    del ents
    _free()
    ents = _rank_entries(m, world, fs[1], m._class_key(None, True, root=True))
    _run_ranks(m, ents, fs[1])
    assert _same(ents[0][4][0], want[1][0]) and _same(ents[0][4][1].view(torch.float16), want[1][1])
    assert all(e[4] is None for e in ents[1:])
    assert [op.name for op in ents[0][0].ops].count("gather_root") == 2
    del ents, m
    _free()


# ---- model files ---------------------------------------------------------------------------------------------------
def _header(path):
    """(flags, class-map role length, map bytes) of a model file"""
    data = open(path, "rb").read(2048)
    flags = struct.unpack_from("<I", data, 8 + 16)[0]
    X, Y, Z = struct.unpack_from("<3I", data, 8 + 36 + 12)
    roles_at = 8 + 36 + 28 + 512 + 56 + 8 + 256 + 20 + 12 + 64 + 4
    return flags, struct.unpack_from("<iQQ", data, roles_at + 7 * 20)[2], X * Y * Z * 2


@pytest.mark.parametrize("name,precision", [(n, p) for n in RELEASED for p in ("tf32", "bf16")] +
                         [("kitti_b7_f64_flosp_a100", "tf32")])
def test_model_file_conf(name, precision, tmp_path):
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    frames = _camera_frames(sc, sc.CONFIGS[name])
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=True) for f in frames]
        deploy.export(m, tmp_path / "conf.occd", frames[0], confidence=True)
        deploy.export(m, tmp_path / "plain.occd", frames[0])
    flags, role, map_bytes = _header(tmp_path / "conf.occd")
    assert flags & 4 and role == 2 * map_bytes
    flags, role, map_bytes = _header(tmp_path / "plain.occd")
    assert not flags & 4 and role == map_bytes
    cm = deploy.LoadedModel(tmp_path / "conf.occd")
    for graph in (True, False):
        for i, (f, (wmap, wconf)) in enumerate(zip(frames, want)):
            cmap, conf = cm.run_frame(f, graph=graph, conf=True)
            torch.cuda.synchronize()
            assert _same(cmap, wmap) and _same(conf, wconf), (graph, i)
            assert _same(cm.run_frame(f, graph=graph), wmap)
    cm.close()
    plain = deploy.LoadedModel(tmp_path / "plain.occd")
    out = torch.empty(want[0][0].shape, dtype=torch.uint16, device="cuda")
    conf = torch.empty(want[0][0].shape, dtype=torch.float16, device="cuda")
    f = _lib.Frame()
    img = torch.as_tensor(frames[0]["img"]).cuda()
    f.images = img.data_ptr()
    rc = _lib.lib().occd_model_run_frame_conf(plain.handle, C.byref(f), out.data_ptr(), conf.data_ptr(), None)
    assert rc == _lib.ERR_UNSUPPORTED and b"without confidence" in _lib.lib().occd_last_error()
    plain.close()
    del m
    _free()
