"""Batched camera frames (OccDepth.predict_frames, CameraPipeline(batch=), batched model files): every frame of a batch
bit for bit what predict_frame gives for that frame alone -- class map, confidence and every logit -- for every shipped
configuration; the per-item virtual view; the per-item calibration cache; the B-frame plan run with a short list; and
batched model files replayed from C (occd_model_run_frames, tools/occd_run)."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200 import data as D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402


def _sc():
    import shipped_configs
    return shipped_configs


def _bits(t):
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def _same(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


# ---- 1. the virtual view with one depth map per item --------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_virtual_view_items(precision):
    L = _lib.lib()
    dt = torch.float32 if precision == "tf32" else torch.bfloat16
    ldt = _lib.DTYPE_F32 if precision == "tf32" else _lib.DTYPE_BF16
    g = torch.Generator(device="cuda").manual_seed(0)
    B, h, w, Cn, cs, dh, dw = 3, 15, 20, 20, 24, 48, 64
    x = torch.randn(B, h, w, cs, device="cuda", generator=g).to(dt)
    pad = 7                                       # a stride larger than one map
    depth = (torch.rand(B, dh * dw + pad, device="cuda", generator=g) * 7.5 + 0.5).contiguous()
    depth[:, ::97] = 0.0                          # inf disparities -> 0
    st = _lib.stream_ptr()

    def run(fn, *a):
        out = torch.full((B, h, w, cs), float("nan"), device="cuda", dtype=dt)
        _lib.check(fn(x.data_ptr(), out.data_ptr(), *a[:1], ldt, B, h, w, Cn, cs, cs, dh, dw, *a[1:], st), "vv")
        return out

    ref0 = run(L.occd_virtual_view_fwd, depth.data_ptr(), 12.5)
    items0 = run(L.occd_virtual_view_items_fwd, depth.data_ptr(), 12.5, 0)
    assert _same(items0, ref0)                    # stride 0 is today's entry point, byte for byte
    per = run(L.occd_virtual_view_items_fwd, depth.data_ptr(), 12.5, dh * dw + pad)
    for b in range(B):
        one = torch.full((1, h, w, cs), float("nan"), device="cuda", dtype=dt)
        _lib.check(L.occd_virtual_view_fwd(x[b].data_ptr(), one.data_ptr(), depth[b].data_ptr(), ldt, 1, h, w, Cn, cs,
                                           cs, dh, dw, 12.5, st), "vv")
        assert _same(per[b:b + 1], one), b
    assert not _same(per[1:2], ref0[1:2])         # item 1 did not read item 0's map


# ---- 2. every shipped configuration: each frame of a batch equals predict_frame of that frame -----------------------
def _kitti_frames(V, hw, full, seeds, shifts):
    geo = kitti_geometry(hw[0], hw[1], full)
    out = []
    for i, (s, sh) in enumerate(zip(seeds, shifts)):
        f = dict(kitti_frame(V, hw[0], hw[1], s, shift=sh), **geo)
        if i == 1:                                # a larger raw image: each frame is staged from its own size
            f["img"] = np.random.default_rng(s).integers(0, 256, size=(V, hw[0] + 9, hw[1] + 14, 3), dtype=np.uint8)
        out.append(f)
    return out


def _nyu_frames(hw, seeds):
    out = []
    for i, s in enumerate(seeds):
        f = nyu_frame(s)
        d = np.array([[0, 0, 0], [0.25, -0.5, 0.125], [-0.25, 0.125, 0.0]][i % 3], float)
        f["vox_origin"] = f["vox_origin"] + d
        f["cam_pose"] = f["cam_pose"].copy()
        f["cam_pose"][:3, 3] += d + np.array([0.1 * i, 0, 0])
        f["img_hw"] = hw
        out.append(f)
    return out


def _check_logits(got, want, i):
    keys = [k for k, v in want.items() if isinstance(v, torch.Tensor)]
    assert keys
    for k in keys:
        assert _same(got[k][i:i + 1], want[k]), (k, i)


CASES = [(n, "tf32") for n in _sc().CONFIGS] + [("nyu_b4_f100_2080ti", "bf16"), ("kitti_b3_f32_flospdepth_2080ti", "bf16")]


@pytest.mark.parametrize("name,precision", CASES)
def test_shipped_config_frame_batches(name, precision, monkeypatch):
    sc = _sc()
    gc.collect()
    torch.cuda.empty_cache()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    nyu = sc.CONFIGS[name]["dataset"] == "NYU"
    V = sc.CONFIGS[name]["views"]
    if nyu:
        frames = _nyu_frames(sc.NYU_IMG, [1, 2, 3])
        again = _nyu_frames(sc.NYU_IMG, [4, 5, 6])
    else:
        # two calibrations; `again` repeats each item's calibration with new images
        frames = _kitti_frames(V, sc.KITTI_IMG, sc.KITTI_FULL, [1, 2, 3], [0.0, 0.3, 0.0])
        again = _kitti_frames(V, sc.KITTI_IMG, sc.KITTI_FULL, [4, 5, 6], [0.0, 0.3, 0.0])
    # the forward plan (every output kept) of the EfficientNet-B7 KITTI configurations takes over 26 GB per frame: at
    # B = 3 it does not fit on an 80 GB card, so their logits are compared at B = 2 (their class maps at 2 and 3)
    logit_batches = (2,) if name.startswith("kitti_b7") else (2, 3)
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=True) for f in frames + again]
        want_logits = [m.predict_frame(f, classes=False) for f in frames]
        for B in (2, 3):
            # the class-map and forward plans are cached side by side: hold one B-frame plan at a time
            m.invalidate_plans()
            got_map, got_conf = m.predict_frames(frames[:B], confidence=True)
            assert got_map.shape[0] == B and got_conf.shape[0] == B
            for i in range(B):
                assert _same(got_map[i:i + 1], want[i][0]), (B, i, int((got_map[i:i + 1] != want[i][0]).sum()))
                assert _same(got_conf[i:i + 1], want[i][1]), (B, i)
            if B == 3:
                calls = []
                orig = D.vox2pix_into
                monkeypatch.setattr(D, "vox2pix_into", lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
                got_map, got_conf = m.predict_frames(again, confidence=True)
                monkeypatch.setattr(D, "vox2pix_into", orig)
                # KITTI: every item keeps its calibration, so no index is recomputed; NYU poses change every frame
                assert len(calls) == (3 * (2 if m.dataset == "NYU" else 0)), len(calls)
                for i in range(3):
                    assert _same(got_map[i:i + 1], want[3 + i][0]), ("again", i)
                    assert _same(got_conf[i:i + 1], want[3 + i][1]), ("again", i)
            if B not in logit_batches:
                continue
            m.invalidate_plans()
            got = m.predict_frames(frames[:B], classes=False)
            for i in range(B):
                _check_logits(got, want_logits[i], i)
            del got
    del m
    gc.collect()
    torch.cuda.empty_cache()


# ---- 3. CameraPipeline(batch=3) over 7 frames -------------------------------------------------------------------------
def _small_kitti():
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    seeds = list(range(1, 8))
    frames = _kitti_frames(2, hw, full, seeds, [0.0, 0.3, 0.0, 0.3, 0.3, 0.0, 0.0])
    return m.cuda(), frames, hw


def _small_nyu():
    sc = _sc()
    hw = (96, 128)
    m, _, _ = sc.make_case("nyu_b4_f100_2080ti", img_hw=hw)
    return m.cuda(), _nyu_frames(hw, list(range(1, 8))), hw


@pytest.mark.parametrize("confidence", [False, True])
def test_camera_pipeline_batch(confidence):
    from occdepth_b200.serving import CameraPipeline
    m, frames, hw = _small_kitti()
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=confidence) for f in frames]
    pipe = CameraPipeline(m, img_hw=hw, vox_origin=frames[0]["vox_origin"], voxel_size=frames[0]["voxel_size"],
                          scene_size=frames[0]["scene_size"], batch=3, confidence=confidence)
    host = [{k: v for k, v in f.items() if k not in ("img_hw", "vox_origin", "voxel_size", "scene_size")}
            for f in frames]
    groups = [host[0:3], host[3:6], host[6:7]]
    got = []
    plan_ids = []
    for grp in groups:
        t = pipe.submit(grp)
        plan_ids.append(id(next(iter(m._class_plans().values()))[0]))
        if t is not None:          # host views, valid until two more submits: keep copies
            r = pipe.result(t)
            got.append(tuple(x.clone() for x in r) if confidence else r.clone())
    r = pipe.result(pipe.flush())
    got.append(tuple(x.clone() for x in r) if confidence else r.clone())
    assert len(set(plan_ids)) == 1                # the short last list runs the same 3-frame plan
    flat = []
    for r, grp in zip(got, groups):
        maps = r[0] if confidence else r
        assert maps.shape[0] == len(grp) and not maps.is_cuda
        for i in range(len(grp)):
            flat.append((maps[i:i + 1], r[1][i:i + 1]) if confidence else maps[i:i + 1])
    assert len(flat) == 7
    for i, (g, w) in enumerate(zip(flat, want)):
        if confidence:
            assert _same(g[0], w[0].cpu()) and _same(g[1], w[1].cpu()), i
        else:
            assert _same(g, w.cpu()), i


# ---- 4. batched model files ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["kitti", "nyu"])
def test_batched_model_file(which, tmp_path):
    m, frames, hw = _small_kitti() if which == "kitti" else _small_nyu()
    frames = frames[:4]
    with torch.no_grad():
        want = [m.predict_frame(f, confidence=True) for f in frames]
        deploy.export(m, tmp_path / "one_a.occd", frames[0])
        deploy.export(m, tmp_path / "b3.occd", frames[:3], confidence=True)
        want3 = m.predict_frames(frames[:3], confidence=True)
    # a single frame dict writes an unbatched file: no flag bit 5, no batch block
    flags = int.from_bytes((tmp_path / "one_a.occd").read_bytes()[24:28], "little")
    assert not flags & deploy.FLAG_BATCH
    assert int.from_bytes((tmp_path / "b3.occd").read_bytes()[24:28], "little") & deploy.FLAG_BATCH
    for i in range(3):
        assert _same(want3[0][i:i + 1], want[i][0]) and _same(want3[1][i:i + 1], want[i][1]), i
    one = deploy.LoadedModel(tmp_path / "one_a.occd")
    assert one.batch() == 1
    one.close()
    cm = deploy.LoadedModel(tmp_path / "b3.occd")
    assert cm.batch() == 3
    side = torch.cuda.Stream()
    for graph in (True, False, True):
        mp, cf = cm.run_frames(frames[:3], stream=side, graph=graph, conf=True)
        side.synchronize()
        assert _same(mp, want3[0]) and _same(cf, want3[1]), graph
        mp = cm.run_frames(frames[3:4], stream=side, graph=graph)          # n = 1 through the 3-frame plan
        side.synchronize()
        assert _same(mp, want[3][0]), graph
        single = cm.run_frame(frames[0], stream=side, graph=graph)        # occd_model_run_frame: n = 1
        side.synchronize()
        assert _same(single, want[0][0]), graph
    with pytest.raises(RuntimeError, match="1 to 3"):
        cm.run_frames(frames[:4])
    cm.close()
    if which == "kitti":
        _check_occd_run(tmp_path / "b3.occd", frames, [w[0] for w in want], tmp_path)
    plain = deploy.LoadedModel(tmp_path / "one_a.occd")
    with pytest.raises(RuntimeError, match="without confidence"):
        plain.run_frames(frames[:1], conf=True)
    plain.close()


def test_export_releases_plans_finalized_while_recording(tmp_path, monkeypatch):
    """a convolution plan of another Plan, left as cyclic garbage, is finalized by a collection inside the recording
    run: the export releases it and writes the model file"""
    from occdepth_b200.engine import CL, FnOp, Plan
    m, frames, _ = _small_kitti()
    dec = m.net_3d_decoder
    orig = type(dec).emit

    def emit(self, plan, x3d, **k):
        out = orig(self, plan, x3d, **k)
        plan.add(FnOp(lambda st: (gc.collect(), 0)[1], "collect"))
        return out
    monkeypatch.setattr(type(dec), "emit", emit)
    gc.collect()
    gc.disable()
    try:
        p = Plan(torch.device("cuda"), precision="tf32")
        x = CL.from_planar(torch.randn(1, 8, 4, 8, 8, device="cuda"), precision="tf32")
        p.conv(x, torch.randn(8, 8, 1, 1, 1, device="cuda"), torch.zeros(8, device="cuda"), act="none")
        p.cycle = p                               # only the collector frees it
        del p, x
        with torch.no_grad():
            info = deploy.export(m, tmp_path / "m.occd", frames[0])
    finally:
        gc.enable()
    assert info["records"] > 0 and (tmp_path / "m.occd").exists()
    with torch.no_grad():
        want = m.predict_frame(frames[0])
    cm = deploy.LoadedModel(tmp_path / "m.occd")
    got = cm.run_frame(frames[0])
    torch.cuda.synchronize()
    assert _same(got, want)
    cm.close()


def _check_occd_run(model_path, frames, want, tmp_path):
    """tools/occd_run on a 3-frame file and 4 frames: a group of 3 and a short group of 1"""
    exe = _build.occd_run_path()
    H0, W0 = max(f["img"].shape[1] for f in frames), max(f["img"].shape[2] for f in frames)
    with open(tmp_path / "imgs.u8", "wb") as fi, open(tmp_path / "calib.f64", "wb") as fc:
        for f in frames:
            img = np.zeros((f["img"].shape[0], H0, W0, 3), np.uint8)
            img[:, :f["img"].shape[1], :f["img"].shape[2]] = f["img"]
            fi.write(img.tobytes())
            fc.write(np.ascontiguousarray(f["cam_k"], np.float64).tobytes())
            fc.write(np.ascontiguousarray(f["T_velo_2_cam"], np.float64).tobytes())
    out = tmp_path / "labels"
    out.mkdir()
    r = subprocess.run([exe, str(model_path), str(tmp_path / "imgs.u8"), str(tmp_path / "calib.f64"),
                        str(len(frames)), str(out), "--raw", str(H0), str(W0)], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "frames 0..2" in r.stdout and "frames 3..3" in r.stdout and "ms per frame" in r.stdout, r.stdout
    for i, w in enumerate(want):
        assert (out / ("%06d.label" % i)).read_bytes() == w.cpu().numpy().tobytes(), i
