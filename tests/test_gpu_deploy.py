"""Model files (occdepth_b200.deploy.export) replayed by the C runtime (occd_model_load / occd_model_run_frame): every
shipped configuration's class maps bit for bit equal to OccDepth.predict_frame of the same frames, with and without
the CUDA graph and the label remap, on a non-default stream; the export's refusals; two models at once; the device
memory a model holds; and tools/occd_run, the standalone C consumer."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402


def _sc():
    import shipped_configs
    return shipped_configs


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _frames(m, spec_views, nyu, hw, full):
    """three frames of different images: KITTI's third changes the calibration, every NYU frame pose and depth"""
    if nyu:
        geo = dict(img_hw=hw)
        frames = [nyu_frame(1 + i) for i in range(3)]
        for i, f in enumerate(frames):
            f["cam_pose"] = f["cam_pose"].copy()
            f["cam_pose"][0, 3] += 0.15 * i
    else:
        geo = kitti_geometry(hw[0], hw[1], full)
        frames = [kitti_frame(spec_views, hw[0], hw[1], 1), kitti_frame(spec_views, hw[0], hw[1], 2),
                  kitti_frame(spec_views, hw[0], hw[1], 3, shift=0.3)]
    return [dict(f, **geo) for f in frames]


CASES = [(n, "tf32") for n in _sc().CONFIGS] + [("nyu_b4_f100_2080ti", "bf16"), ("kitti_b3_f32_flospdepth_2080ti", "bf16")]
RELEASED_KITTI = "kitti_b3_f32_flospdepth_2080ti"


@pytest.mark.parametrize("name,precision", CASES)
def test_shipped_config_model_file_parity(name, precision, tmp_path):
    sc = _sc()
    gc.collect()
    torch.cuda.empty_cache()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    nyu = sc.CONFIGS[name]["dataset"] == "NYU"
    frames = _frames(m, sc.CONFIGS[name]["views"], nyu, sc.NYU_IMG if nyu else sc.KITTI_IMG, sc.KITTI_FULL)
    inv = np.random.default_rng(3).permutation(256)[:m.n_classes]
    with torch.no_grad():
        want = [m.predict_frame(f) for f in frames]
        want_inv = [m.predict_frame(f, inv_map=inv) for f in frames]
        deploy.export(m, tmp_path / "plain.occd", frames[0])
        deploy.export(m, tmp_path / "inv.occd", frames[0], inv_map=inv)
    side = torch.cuda.Stream()
    for path, w in ((tmp_path / "plain.occd", want), (tmp_path / "inv.occd", want_inv)):
        cm = deploy.LoadedModel(path)
        # graph: the first frame captures, the others replay it; then one by one; then the graph again
        for graph in (True, False, True):
            got = [cm.run_frame(f, stream=side, graph=graph) for f in frames]
            side.synchronize()
            for i, (g, x) in enumerate(zip(got, w)):
                assert _same(g, x), (path.name, graph, i, int((g.int() != x.int()).sum()))
        assert cm.info().graph == 1
        cm.close()
    if name == RELEASED_KITTI and precision == "tf32":
        _check_occd_run(tmp_path / "inv.occd", frames, want_inv, tmp_path)
    del m
    gc.collect()
    torch.cuda.empty_cache()


def _check_occd_run(model_path, frames, want, tmp_path):
    """tools/occd_run on raw image and calibration files writes the same .label bytes as predict_frame's maps"""
    exe = _build.occd_run_path()
    H0, W0 = frames[0]["img"].shape[1:3]
    with open(tmp_path / "imgs.u8", "wb") as fi, open(tmp_path / "calib.f64", "wb") as fc:
        for f in frames:
            fi.write(np.ascontiguousarray(f["img"], np.uint8).tobytes())
            fc.write(np.ascontiguousarray(f["cam_k"], np.float64).tobytes())
            fc.write(np.ascontiguousarray(f["T_velo_2_cam"], np.float64).tobytes())
    out = tmp_path / "labels"
    out.mkdir()
    r = subprocess.run([exe, str(model_path), str(tmp_path / "imgs.u8"), str(tmp_path / "calib.f64"),
                        str(len(frames)), str(out), "--raw", str(H0), str(W0)], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ms per frame" in r.stdout
    for i, w in enumerate(want):
        assert (out / ("%06d.label" % i)).read_bytes() == w.cpu().numpy().tobytes(), i


def test_nyu_flosp_depth_model_file_parity(tmp_path):
    """NYU with the FlospDepth prior (no shipped configuration runs it): FlospDepth's grid is re-derived from every
    frame's origin in its own axis order, and a float32 pose without cam_k takes the default intrinsics in float32"""
    sc = _sc()
    spec = dict(dataset="NYU", backbone_2d_name="tf_efficientnet_b3_ns", feature=16, trans_2d_to_3d="flosp_depth",
                views=1, context_prior=False, cascade_cls=False, use_depth_gt=True)
    m, _, _ = sc.make_case(spec=spec)               # the NYU grid FlospDepth's bounds give: 60 x 36 x 60 voxels
    m = m.cuda()
    frames = _frames(m, 1, True, sc.NYU_IMG, None)
    f32 = dict(frames[2], cam_pose=frames[2]["cam_pose"].astype(np.float32))
    del f32["cam_k"]
    frames.append(f32)
    with torch.no_grad():
        want = [m.predict_frame(f) for f in frames]
        deploy.export(m, tmp_path / "nyu.occd", frames[0])
    side = torch.cuda.Stream()
    cm = deploy.LoadedModel(tmp_path / "nyu.occd")
    for graph in (True, False):
        got = [cm.run_frame(f, stream=side, graph=graph) for f in frames]
        side.synchronize()
        for i, (g, w) in enumerate(zip(got, want)):
            assert _same(g, w), (graph, i, int((g.int() != w.int()).sum()))
    cm.close()


def _small(name="kitti_b3_f32_flospdepth_2080ti", **k):
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, _, _ = sc.make_case(name, img_hw=hw, full=full, **k)
    return m.cuda(), _frames(m, sc.CONFIGS[name]["views"], False, hw, full)


def test_export_refusals(tmp_path):
    from occdepth_b200.parallel import SimSlabGroup
    m, frames = _small()
    f = frames[0]
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="one frame"):
            deploy.export(m, tmp_path / "x.occd", dict(f, img=np.stack([f["img"]] * 2)))
        m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        try:
            with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
                deploy.export(m, tmp_path / "x.occd", f)
        finally:
            m.__dict__.pop("slab_ctx", None)
        mi, _ = _small(infer_mode=True)
        with pytest.raises(NotImplementedError, match="infer_mode"):
            deploy.export(mi, tmp_path / "x.occd", f)
    assert not (tmp_path / "x.occd").exists()


def test_export_refuses_a_pointer_it_cannot_place(tmp_path, monkeypatch):
    """a launch whose closure reads a tensor the plan does not hold: the export names the entry point and argument"""
    from occdepth_b200.engine import FnOp
    m, frames = _small()
    dec = m.net_3d_decoder
    orig = type(dec).emit
    stray = torch.zeros(64, device="cuda")

    def emit(self, plan, x3d, **k):
        out = orig(self, plan, x3d, **k)
        L = _lib.lib()
        plan.add(FnOp(lambda st: L.occd_softmax_planar(stray.data_ptr(), out.data_ptr(), 1, 1, 1, st), "stray"))
        return out
    monkeypatch.setattr(type(dec), "emit", emit)
    with torch.no_grad(), pytest.raises(deploy.ExportError, match="occd_softmax_planar argument 0"):
        deploy.export(m, tmp_path / "x.occd", frames[0])


def test_two_models_and_device_memory(tmp_path):
    m1, fr1 = _small()
    m2, _ = _small("kitti_b7_f64_flosp_a100")
    with torch.no_grad():
        deploy.export(m1, tmp_path / "a.occd", fr1[0])
        deploy.export(m2.set_precision("bf16"), tmp_path / "b.occd", fr1[0])
    side = torch.cuda.Stream()

    def run_all(cm):
        r = [cm.run_frame(f, stream=side) for f in fr1]
        side.synchronize()
        return r
    alone = []
    for p in ("a.occd", "b.occd"):
        cm = deploy.LoadedModel(tmp_path / p)
        alone.append(run_all(cm))
        cm.close()
    a, b = deploy.LoadedModel(tmp_path / "a.occd"), deploy.LoadedModel(tmp_path / "b.occd")
    for i, f in enumerate(fr1):                   # interleaved: each model keeps its own calibration and graph
        ga, gb = a.run_frame(f, stream=side), b.run_frame(f, stream=side)
        side.synchronize()
        assert _same(ga, alone[0][i]) and _same(gb, alone[1][i]), i
    a.close()
    b.close()
    # the memory a model holds: what info reports comes back on destroy (driver granularity 2 MB)
    out = torch.empty(1, 64, 64, 16, dtype=torch.uint16, device="cuda")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    cm = deploy.LoadedModel(tmp_path / "a.occd")
    for f in fr1:
        cm.run_frame(f, out=out)
    torch.cuda.synchronize()
    held = cm.info().device_bytes
    free1 = torch.cuda.mem_get_info()[0]
    cm.close()
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    assert held > 0
    assert abs((free0 - free1) - held) <= 2 << 20, (free0 - free1, held)
    assert abs((free2 - free1) - held) <= 2 << 20, (free2 - free1, held)
