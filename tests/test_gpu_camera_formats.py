"""Camera frames in the formats cameras and video decoders deliver (BGR, NV12) and from unrectified cameras
(per-view maps of cv2.initUndistortRectifyMap): the staging kernel against its host emulation, and every route --
predict_frame, predict_frames, CameraPipeline, the X-slab partition, model files and tools/occd_run -- bit for bit
what the same route gives for the RGB frame OpenCV makes from the same input on the host."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200 import data as D

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402
from test_stage_camera_host import emul  # noqa: E402,F401  (the host emulation's build, shared)

DIST = np.array([-0.22, 0.06, 0.0008, -0.0011, 0.0])


def _sc():
    import shipped_configs
    return shipped_configs


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


def _own(r):
    """a copy of a result: a map, (map, conf) or the forward's dict may live in the plan's buffers"""
    if isinstance(r, dict):
        return {k: v.clone() for k, v in r.items() if isinstance(v, torch.Tensor)}
    return tuple(x.clone() for x in r) if isinstance(r, tuple) else r.clone()


def _free():
    gc.collect()
    torch.cuda.empty_cache()


# ---- what a camera delivers, and the RGB frame OpenCV makes of it on the host ---------------------------------------
def _nv12(g, V, H0, W0):
    return g.integers(0, 256, size=(V, H0 * 3 // 2, W0), dtype=np.uint8)


def _nv12_h(H0):
    """an even luma height at least H0 that is 2 mod 4 (as KITTI's raw 370 and 374 rows are): half of it is odd"""
    h = H0 + H0 % 2
    return h + 2 if h % 4 == 0 else h


def _maps(cam_k, H, W):
    """per view the x, y maps that undistort a camera with cam_k and DIST into the pinhole cam_k, at the crop size"""
    out = []
    for K in np.asarray(cam_k).reshape(-1, 3, 3):
        mx, my = cv2.initUndistortRectifyMap(K, DIST, None, K, (W, H), cv2.CV_32FC1)
        out.append(np.stack([mx, my]))
    return np.stack(out).astype(np.float32)


def _host_rgb(img, fmt, maps=None):
    """OpenCV's host route: cvtColor, then remap -> uint8 RGB (V, h, w, 3)"""
    code = {"bgr": cv2.COLOR_BGR2RGB, "nv12": cv2.COLOR_YUV2RGB_NV12}[fmt]
    rgb = [cv2.cvtColor(np.ascontiguousarray(im), code) for im in img]
    if maps is not None:
        rgb = [cv2.remap(r, m[0], m[1], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
               for r, m in zip(rgb, maps)]
    return np.stack(rgb)


def _variants(frame, seed):
    """(device-format frame, the RGB frame OpenCV makes of it) for BGR, NV12 and NV12 with rectification maps"""
    g = np.random.default_rng(seed)
    V, H0, W0 = frame["img"].shape[:3]
    H, W = frame["img_hw"]
    cam_k = frame.get("cam_k", np.array([[518.8579, 0, 320], [0, 518.8579, 240], [0, 0, 1]]))
    bgr = np.ascontiguousarray(frame["img"][..., ::-1])
    nv12 = _nv12(g, V, _nv12_h(H0), W0 + W0 % 2)
    maps = _maps(cam_k, H, W)
    return [(dict(frame, img=bgr, pixel_format="bgr"), dict(frame, img=_host_rgb(bgr, "bgr"))),
            (dict(frame, img=nv12, pixel_format="nv12"), dict(frame, img=_host_rgb(nv12, "nv12"))),
            (dict(frame, img=nv12, pixel_format="nv12", rect_maps=maps),
             dict(frame, img=_host_rgb(nv12, "nv12", maps)))]


# ---- 1. the kernel against its host emulation ----------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("fmt,with_maps", [("rgb", True), ("bgr", False), ("bgr", True), ("nv12", False),
                                           ("nv12", True)])
def test_kernel_matches_emulation(emul, precision, fmt, with_maps):
    g = np.random.default_rng(11)
    n, H0, W0, H, W, cs = 3, 94, 162, 87, 151, 16
    if fmt == "nv12":
        img = torch.from_numpy(_nv12(g, n, H0, W0))
    else:
        img = torch.from_numpy(g.integers(0, 256, size=(n, H0, W0, 3), dtype=np.uint8))
    maps = None
    if with_maps:
        K = np.array([[120.0, 0, 80], [0, 120.0, 45], [0, 0, 1]])
        maps = np.stack([_maps(K, H, W)[0] + g.normal(0, 3, size=(2, H, W)).astype(np.float32) for _ in range(n)])
        maps[0, 0, 5, 7], maps[1, 1, 9, 2], maps[2, 0, 3, 3] = np.nan, np.inf, -1e30
    dt, ldt = (torch.float32, _lib.DTYPE_F32) if precision == "tf32" else (torch.bfloat16, _lib.DTYPE_BF16)
    out = torch.full((n, H, W, cs), float("nan"), dtype=dt, device="cuda")
    D.stage_camera_u8(img.cuda(), out, ldt, H, W, fmt, None if maps is None else torch.from_numpy(maps).cuda())
    want = torch.empty(out.shape, dtype=dt)
    m, s = np.asarray(D.IMAGENET_MEAN, np.float32), np.asarray(D.IMAGENET_STD, np.float32)
    imgc = np.ascontiguousarray(img.numpy())
    mp = None if maps is None else np.ascontiguousarray(maps)
    rs = W0 if fmt == "nv12" else W0 * 3
    assert emul.stage_camera_emulate(imgc.ctypes.data, _lib.PIXEL_FORMATS[fmt], imgc[0].nbytes, rs, H0 * W0, n, H0,
                                     W0, H, W, None if mp is None else mp.ctypes.data, 2 * H * W, m.ctypes.data,
                                     s.ctypes.data, want.data_ptr(), ldt, cs) == 0
    torch.cuda.synchronize()
    assert _same(out.cpu(), want)


# ---- 2. every shipped configuration: a camera-format frame gives the RGB frame's map, confidence and logits ----------
CASES = [(n, "tf32") for n in _sc().CONFIGS] + [("nyu_b4_f100_2080ti", "bf16"),
                                                 ("kitti_b3_f32_flospdepth_2080ti", "bf16")]


def _frame(sc, name, seed):
    spec = sc.CONFIGS[name]
    if spec["dataset"] == "NYU":
        return dict(nyu_frame(seed), img_hw=sc.NYU_IMG)
    H, W = sc.KITTI_IMG
    return dict(kitti_frame(spec["views"], H, W, seed), **kitti_geometry(H, W, sc.KITTI_FULL))


@pytest.mark.parametrize("name,precision", CASES)
def test_shipped_config_formats(name, precision):
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    with torch.no_grad():
        for k, (cam, ref) in enumerate(_variants(_frame(sc, name, 1), 7)):
            want = _own(m.predict_frame(ref, confidence=True))
            got = m.predict_frame(cam, confidence=True)
            assert _same(got[0], want[0]) and _same(got[1], want[1]), (name, k)
            want = _own(m.predict_frame(ref, classes=False))
            got = m.predict_frame(cam, classes=False)
            keys = list(want)
            assert keys and all(_same(got[key], want[key]) for key in keys), (name, k)
            del want, got
    del m
    _free()


# ---- 3. predict_frames, CameraPipeline, the slab partition, model files: the small KITTI model --------------------
def _small_kitti():
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    frames = [dict(kitti_frame(2, hw[0], hw[1], s, shift=0.3 * (s % 2)), **kitti_geometry(hw[0], hw[1], full))
              for s in (1, 2, 3)]
    return m.cuda(), frames, hw


def test_predict_frames_mixed_formats():
    m, frames, _ = _small_kitti()
    (bgr, bgr_ref), _, (nv, nv_ref) = _variants(frames[0], 3)
    nv = dict(nv, T_velo_2_cam=frames[1]["T_velo_2_cam"])
    nv_ref = dict(nv_ref, T_velo_2_cam=frames[1]["T_velo_2_cam"])
    with torch.no_grad():
        want = [_own(m.predict_frame(f, confidence=True)) for f in (bgr_ref, nv_ref)]
        want_logits = [_own(m.predict_frame(f, classes=False)) for f in (bgr_ref, nv_ref)]
        got = m.predict_frames([bgr, nv], confidence=True)
        for i in range(2):
            assert _same(got[0][i:i + 1], want[i][0]) and _same(got[1][i:i + 1], want[i][1]), i
        got = m.predict_frames([bgr, nv], classes=False)
        for i in range(2):
            for k, v in want_logits[i].items():
                assert _same(got[k][i:i + 1], v), (k, i)


def test_plan_keys_unchanged():
    m, frames, _ = _small_kitti()
    (bgr, _), _, (nv, _) = _variants(frames[0], 3)
    with torch.no_grad():
        m.predict_frame(frames[0])
        plans = dict(m._class_plans())
        m.predict_frame(bgr)
        m.predict_frame(nv)
        assert dict(m._class_plans()).keys() == plans.keys()


def test_camera_pipeline_nv12():
    from occdepth_b200.serving import CameraPipeline
    m, frames, hw = _small_kitti()
    geo = {k: frames[0][k] for k in ("vox_origin", "voxel_size", "scene_size")}
    variants = [_variants(f, 20 + i) for i, f in enumerate(frames)]
    maps = variants[0][2][0]["rect_maps"]
    strip = ("img_hw", "vox_origin", "voxel_size", "scene_size", "pixel_format", "rect_maps")
    results = {}
    for name, kw, k in (("rgb", {}, 1), ("nv12", dict(pixel_format="nv12"), 1),
                        ("nv12_maps", dict(pixel_format="nv12", rect_maps=maps), 2)):
        pipe = CameraPipeline(m, img_hw=hw, confidence=True, **geo, **kw)
        out, h2d = [], []
        for v in variants:
            cam, ref = v[k]
            f = ref if name == "rgb" else cam
            if name == "nv12_maps":       # every frame of the pipeline carries the rig's maps
                f = dict(cam, rect_maps=maps)
            t = pipe.submit({key: val for key, val in f.items() if key not in strip})
            h2d.append(pipe.h2d_bytes)
            if t is not None:
                out.append(tuple(x.clone() for x in pipe.result(t)))
        out.append(tuple(x.clone() for x in pipe.result(pipe.flush())))
        results[name] = (out, h2d)
    V, H0, W0 = frames[0]["img"].shape[:3]
    H0e, W0e = _nv12_h(H0), W0 + W0 % 2
    assert results["rgb"][1] == [V * H0e * W0e * 3] * 3
    assert results["nv12"][1] == [V * H0e * W0e * 3 // 2] * 3      # half the bytes of the RGB frame
    with torch.no_grad():
        for i, v in enumerate(variants):
            want = m.predict_frame(v[1][1], confidence=True)
            got = results["rgb"][0][i]
            assert _same(got[0], want[0].cpu()) and _same(got[1], want[1].cpu()), i
            assert _same(results["nv12"][0][i][0], want[0].cpu()), i
            want = m.predict_frame(dict(v[2][1], img=_host_rgb(v[2][0]["img"], "nv12", maps)), confidence=True)
            got = results["nv12_maps"][0][i]
            assert _same(got[0], want[0].cpu()) and _same(got[1], want[1].cpu()), i


def test_slab_lockstep_view_sharding(monkeypatch):
    """two ranks, each staging its own view with that view's maps, in lock step on one GPU"""
    from occdepth_b200.parallel import SimSlabGroup
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    m, frames, _ = _small_kitti()
    _, _, (cam, ref) = _variants(frames[0], 5)
    with torch.no_grad():
        want = m.predict_frame(ref).clone()
    m.invalidate_plans()
    dev = next(m.parameters()).device
    f = m._frame_inputs(cam, dev)
    grp = SimSlabGroup(2, halo=3)
    ents = []
    try:
        for r in range(2):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad(), torch.cuda.device(dev):
                ents.append(m._build(1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["batch"],
                                     classes=("classes", None)))
    finally:
        m.__dict__.pop("slab_ctx", None)
    assert [e[7] for e in ents] == [0, 1]            # view sharding: rank r stages view r
    for e in ents:
        m._stage_frame(e, f)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    torch.cuda.synchronize()
    assert _same(torch.cat([e[4] for e in ents], 1), want)


def test_model_files(tmp_path):
    m, frames, hw = _small_kitti()
    variants = [_variants(f, 30 + i) for i, f in enumerate(frames)]
    maps = variants[0][2][0]["rect_maps"]
    nv12 = [v[1][0] for v in variants]                               # NV12 frames without maps
    with torch.no_grad():
        deploy.export(m, tmp_path / "plain.occd", frames[0])
        deploy.export(m, tmp_path / "maps.occd", dict(nv12[0], rect_maps=maps), confidence=True)
        want_plain = [_own(m.predict_frame(v[1][1])) for v in variants]
        want_maps = [_own(m.predict_frame(dict(v[1][1], img=_host_rgb(v[1][0]["img"], "nv12", maps)),
                                          confidence=True)) for v in variants]
    flags = lambda p: int.from_bytes((tmp_path / p).read_bytes()[24:28], "little")    # noqa: E731
    assert not flags("plain.occd") & deploy.FLAG_MAPS and flags("maps.occd") & deploy.FLAG_MAPS
    plain, rect = deploy.LoadedModel(tmp_path / "plain.occd"), deploy.LoadedModel(tmp_path / "maps.occd")
    for graph in (True, False):
        for i, v in enumerate(variants):
            got = plain.run_frames([v[1][0]], graph=graph, pixel_format="nv12")
            torch.cuda.synchronize()
            assert _same(got, want_plain[i]), (graph, i)
            got = plain.run_frame(v[1][1], graph=graph)                # RGB through the unchanged entry point
            torch.cuda.synchronize()
            assert _same(got, want_plain[i]), (graph, i)
            mp, cf = rect.run_frames([v[1][0]], graph=graph, conf=True)      # the frame's own "nv12"
            torch.cuda.synchronize()
            assert _same(mp, want_maps[i][0]) and _same(cf, want_maps[i][1]), (graph, i)
    plain.close()
    rect.close()
    # tools/occd_run --format nv12 on the file with maps
    exe = _build.occd_run_path()
    with open(tmp_path / "imgs.u8", "wb") as fi, open(tmp_path / "calib.f64", "wb") as fc:
        for f in nv12:
            fi.write(np.ascontiguousarray(f["img"]).tobytes())
            fc.write(np.ascontiguousarray(f["cam_k"], np.float64).tobytes())
            fc.write(np.ascontiguousarray(f["T_velo_2_cam"], np.float64).tobytes())
    out = tmp_path / "labels"
    out.mkdir()
    V, h, W0 = nv12[0]["img"].shape
    r = subprocess.run([exe, str(tmp_path / "maps.occd"), str(tmp_path / "imgs.u8"), str(tmp_path / "calib.f64"),
                        str(len(nv12)), str(out), "--raw", str(h * 2 // 3), str(W0), "--format", "nv12"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for i, w in enumerate(want_maps):
        assert (out / ("%06d.label" % i)).read_bytes() == w[0].cpu().numpy().tobytes(), i


def test_batched_export_refuses_different_maps(tmp_path):
    m, frames, _ = _small_kitti()
    (_, _), (nv, _), (nvm, _) = _variants(frames[0], 3)
    with torch.no_grad(), pytest.raises(ValueError, match="rect_maps"):
        deploy.export(m, tmp_path / "b.occd", [nvm, nv])
    with torch.no_grad():
        deploy.export(m, tmp_path / "b.occd", [nvm, dict(nvm)])
    assert int.from_bytes((tmp_path / "b.occd").read_bytes()[24:28], "little") & deploy.FLAG_MAPS
