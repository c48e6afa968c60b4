"""The occupied-voxel list of model files (occd_model_list_voxels, LoadedModel.list_voxels) and of lists of camera
frames (OccDepth.predict_voxels([...])): counts, histograms and the written rows of index, cls and xyz bit for bit
those of predict_voxels of the same frames -- the released KITTI and NYU models, label remaps, truncation, a changing
calibration, batched files, NV12 with rectification maps, X-slab files run by a local group -- and tools/occd_run
--voxels."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200.parallel import SimSlabGroup

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402

RELEASED_KITTI, RELEASED_NYU = "kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti"


def _sc():
    import shipped_configs
    return shipped_configs


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _bytes(t):
    return t.contiguous().cpu().numpy().tobytes()


def _same_list(got, want, gb=0, wb=0, what="", keys=("index", "cls", "xyz")):
    """item gb of VoxelList `got` against item wb of `want`: the counts, the histogram and every written row"""
    torch.cuda.synchronize()
    gc_, wc = got.counts()[gb], want.counts()[wb]
    assert gc_.tolist() == wc.tolist(), (what, gc_.tolist(), wc.tolist())
    assert _bytes(got.hist[gb]) == _bytes(want.hist[wb]), what
    n = int(min(wc.sum(), want.capacity))
    assert got.capacity == want.capacity, what
    for k in keys:
        g, w = getattr(got, k), getattr(want, k)
        assert (g is None) == (w is None), (what, k)
        if g is not None:
            assert _bytes(g[gb, :n]) == _bytes(w[wb, :n]), (what, k)
    return gc_


def _kitti_frames(views, hw, full, n=3):
    geo = kitti_geometry(hw[0], hw[1], full)
    return [dict(kitti_frame(views, hw[0], hw[1], 1 + i, shift=0.3 * (i % 2)), **geo) for i in range(n)]


# ---- 1, 2: the released KITTI model from an unbatched file -------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_released_kitti_model_file_lists(precision, tmp_path):
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(RELEASED_KITTI)
    m = m.cuda().set_precision(precision)
    views = sc.CONFIGS[RELEASED_KITTI]["views"]
    A, B = _kitti_frames(views, sc.KITTI_IMG, sc.KITTI_FULL, 2)
    A2 = dict(A, img=kitti_frame(views, sc.KITTI_IMG[0], sc.KITTI_IMG[1], 9)["img"])    # A's calibration, new images
    inv = np.random.default_rng(3).permutation(np.arange(1, 250))[:m.n_classes]
    inv[0] = 0
    with torch.no_grad():
        deploy.export(m, tmp_path / "plain.occd", A)
        deploy.export(m, tmp_path / "inv.occd", A, inv_map=inv)
    cm = deploy.LoadedModel(tmp_path / "plain.occd")
    side = torch.cuda.Stream()
    # the calibration sequence A, A, B, A, B: the second A and the B after it are run without a listing
    listed = {0: A, 3: A, 4: B}
    with torch.no_grad():
        for i, f in enumerate((A, A2, B, A, B)):
            cm.run_frame(f, stream=side)
            if i not in listed:
                continue
            got = cm.list_voxels(stream=side)
            side.synchronize()
            c = _same_list(got, m.predict_voxels(f), what=(precision, "sequence", i))
            assert c[0] > 0 and c[1] > 0
        # truncated, without coordinates, with an origin
        want = m.predict_voxels(B)
        total = int(want.counts()[0].sum())
        cap = total - 5
        _same_list(cm.list_voxels(capacity=cap), m.predict_voxels(B, capacity=cap), what="truncated")
        assert cm.list_voxels(capacity=cap).truncated
        no_xyz = cm.list_voxels(xyz=False)
        assert no_xyz.xyz is None
        _same_list(no_xyz, want, what="no xyz", keys=("index", "cls"))
        origin = [0.5, -25.6, -2.25]
        _same_list(cm.list_voxels(vox_origin=origin), m.predict_voxels(B, vox_origin=origin), what="origin")
        # out= reuses the tensors
        out = cm.list_voxels()
        assert cm.list_voxels(out=out) is out
        _same_list(out, want, what="out")
    cm.close()
    # the label remap of the file
    ci = deploy.LoadedModel(tmp_path / "inv.occd")
    with torch.no_grad():
        for f in (A, B):
            ci.run_frame(f, graph=False)
            _same_list(ci.list_voxels(), m.predict_voxels(f, inv_map=inv), what=(precision, "inv_map"))
    ci.close()
    del m
    _free()


# ---- 3, 7, 8: small models: batched files, refusals, lists of frames ---------------------------------------------------
def _small_kitti():
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, _, _ = sc.make_case(RELEASED_KITTI, img_hw=hw, full=full)
    return m.cuda(), _kitti_frames(2, hw, full, 4), hw


def _small_nyu():
    sc = _sc()
    hw = (96, 128)
    m, _, _ = sc.make_case(RELEASED_NYU, img_hw=hw)
    frames = []
    for i in range(3):
        f = dict(nyu_frame(1 + i), img_hw=hw)
        f["cam_pose"] = f["cam_pose"].copy()
        f["cam_pose"][0, 3] += 0.15 * i
        frames.append(f)
    return m.cuda(), frames, hw


def test_batched_file_lists_and_refusals(tmp_path):
    m, frames, _ = _small_kitti()
    with torch.no_grad():
        deploy.export(m, tmp_path / "b3.occd", frames[:3])
        singles = [m.predict_voxels(f) for f in frames]
    cm = deploy.LoadedModel(tmp_path / "b3.occd")
    with pytest.raises(RuntimeError, match="no run yet"):
        cm.list_voxels()
    bytes0 = cm.info().device_bytes
    side = torch.cuda.Stream()
    with torch.no_grad():
        for idx in ((2, 1), (0, 1, 2), (3, 0)):
            n, fs = len(idx), [frames[i] for i in idx]
            cm.run_frames(fs, stream=side)
            got = cm.list_voxels(stream=side)
            side.synchronize()
            assert got.B == n
            want = m.predict_voxels(fs)
            assert want.B == n
            for b, i in enumerate(idx):
                _same_list(got, want, b, b, what=(n, b, "list"))
                _same_list(got, singles[i], b, 0, what=(n, b, "single"))
            first = cm.list_voxels(n=1)
            _same_list(first, want, 0, 0, what=(n, "n=1"))
        with pytest.raises(RuntimeError, match="the last run ran 1 to 2"):
            cm.list_voxels(n=3)
    # the scratch: three items' masks and the work array, held from the first listing on
    N = 64 * 64 * 16
    assert cm.info().device_bytes == bytes0 + 3 * N + 4 * _lib.voxel_work_len(3, N)
    cm.close()


@pytest.mark.parametrize("which", ["kitti", "nyu"])
def test_predict_voxels_of_a_list_equals_the_single_lists(which):
    m, frames, _ = _small_kitti() if which == "kitti" else _small_nyu()
    f0, f1 = frames[0], frames[2]
    with torch.no_grad():
        want = [m.predict_voxels(f) for f in (f0, f1)]
        for _ in range(2):                         # the second pass: each position's mask is kept
            got = m.predict_voxels([f0, f1])
            for b in range(2):
                c = _same_list(got, want[b], b, 0, what=(which, b))
                assert c[0] > 0 and (c[1] > 0) == (which == "kitti")
        swapped = m.predict_voxels([f1, f0])      # the positions' calibrations change: their masks follow
        _same_list(swapped, want[1], 0, 0, what=(which, "swapped 0"))
        _same_list(swapped, want[0], 1, 0, what=(which, "swapped 1"))
        # an explicit mask per frame, and the single-frame route still as it was
        if which == "kitti":
            masks = np.random.default_rng(4).random((2, 64 * 64 * 16)) < 0.5
            got = m.predict_voxels([f0, f1], fov_mask=masks, capacity=500)
            for b, f in enumerate((f0, f1)):
                _same_list(got, m.predict_voxels(f, fov_mask=masks[b], capacity=500), b, 0, what=("mask", b))
            with pytest.raises(ValueError, match="1 masks for 2 frames"):
                m.predict_voxels([f0, f1], fov_mask=masks[:1])
        _same_list(m.predict_voxels(f0), want[0], what=(which, "single after"))


# ---- 4: the released NYU model ----------------------------------------------------------------------------------------
def test_released_nyu_model_file_lists(tmp_path):
    sc = _sc()
    _free()
    m, _, _ = sc.make_case(RELEASED_NYU)
    m = m.cuda().set_precision("bf16")
    frames = []
    for i in range(2):
        f = dict(nyu_frame(1 + i), img_hw=sc.NYU_IMG)
        f["cam_pose"] = f["cam_pose"].copy()
        f["cam_pose"][0, 3] += 0.2 * i
        frames.append(f)
    with torch.no_grad():
        deploy.export(m, tmp_path / "nyu.occd", frames[0])
    cm = deploy.LoadedModel(tmp_path / "nyu.occd")
    assert cm.geom.has_depth == 1
    with torch.no_grad():
        for i, f in enumerate(frames):
            cm.run_frame(f)
            c = _same_list(cm.list_voxels(), m.predict_voxels(f), what=("nyu", i))
            assert c[0] > 0 and c[1] == 0            # no mask: every row counts as inside
    cm.close()
    del m
    _free()


# ---- 5: NV12 input with rectification maps ----------------------------------------------------------------------------
def test_nv12_rectified_model_file_lists(tmp_path):
    m, frames, hw = _small_kitti()
    H, W = hw
    g = np.random.default_rng(7)
    V = frames[0]["img"].shape[0]
    ys, xs = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    maps = np.stack([np.stack([xs * 0.97 + 3.3 + v, ys * 0.98 + 1.7]) for v in range(V)]).astype(np.float32)
    nv = [dict(f, img=g.integers(0, 256, size=(V, (H + 2) * 3 // 2, W + 6), dtype=np.uint8), pixel_format="nv12")
          for f in frames[:3]]
    with torch.no_grad():
        deploy.export(m, tmp_path / "nv12.occd", dict(nv[0], rect_maps=maps))
    cm = deploy.LoadedModel(tmp_path / "nv12.occd")
    with torch.no_grad():
        for i, f in enumerate(nv):
            cm.run_frames([f])
            _same_list(cm.list_voxels(), m.predict_voxels(dict(f, rect_maps=maps)), what=("nv12", i))
    cm.close()


# ---- 6: X-slab files run by a local group ------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
def test_slab_files_list_on_rank_0(world, tmp_path):
    sc = _sc()
    hw, full = (96, 320), (128, 128, 16)
    m, _, _ = sc.make_case(RELEASED_KITTI, img_hw=hw, full=full)
    m = m.cuda()
    frames = _kitti_frames(2, hw, full, 3)
    with torch.no_grad():
        want = [m.predict_voxels(f) for f in frames]
    paths = [tmp_path / ("r%d.occd" % r) for r in range(world)]
    grp = SimSlabGroup(world, halo=3)
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                deploy.export(m, paths[r], frames[0], slab_output="root")
    finally:
        m.__dict__.pop("slab_ctx", None)
    comms = deploy.Comm.local(world)
    models = [deploy.LoadedModel(p, c) for p, c in zip(paths, comms)]
    for graph in (True, False):
        for i, f in enumerate(frames):
            deploy.run_frame_group(models, f, graph=graph)
            _same_list(models[0].list_voxels(), want[i], what=(world, graph, i))
    with pytest.raises(RuntimeError, match="rank 1 of the X-slab partition holds no map"):
        models[1].list_voxels()
    for x in models:
        x.close()


# ---- tools/occd_run --voxels ------------------------------------------------------------------------------------------
def test_occd_run_voxels(tmp_path):
    m, frames, _ = _small_kitti()
    frames = frames[:2]
    with torch.no_grad():
        deploy.export(m, tmp_path / "k.occd", frames[0])
    cm = deploy.LoadedModel(tmp_path / "k.occd")
    lists = []
    for f in frames:
        cm.run_frame(f)
        lists.append(cm.list_voxels())
    torch.cuda.synchronize()
    cm.close()
    with open(tmp_path / "imgs.u8", "wb") as fi, open(tmp_path / "calib.f64", "wb") as fc:
        for f in frames:
            fi.write(np.ascontiguousarray(f["img"], np.uint8).tobytes())
            fc.write(np.ascontiguousarray(f["cam_k"], np.float64).tobytes())
            fc.write(np.ascontiguousarray(f["T_velo_2_cam"], np.float64).tobytes())
    out = tmp_path / "labels"
    out.mkdir()
    H0, W0 = frames[0]["img"].shape[1:3]
    cap = int(lists[0].counts()[0].sum()) - 3                # frame 0's list is truncated
    r = subprocess.run([_build.occd_run_path(), str(tmp_path / "k.occd"), str(tmp_path / "imgs.u8"),
                        str(tmp_path / "calib.f64"), str(len(frames)), str(out), "--raw", str(H0), str(W0),
                        "--voxels", str(cap)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for i, vl in enumerate(lists):
        data = (out / ("%06d.voxels" % i)).read_bytes()
        count = np.frombuffer(data, "<i4", 2)
        hist = np.frombuffer(data, "<i4", 64, 8)
        n = int(min(count.sum(), cap))
        assert len(data) == 8 + 256 + 18 * n
        assert count.tolist() == vl.counts()[0].tolist(), i
        assert "frame %d: %d voxels inside the FOV, %d outside" % (i, count[0], count[1]) in r.stdout
        assert hist.tobytes() == _bytes(vl.hist[0]), i
        o = 8 + 256
        assert data[o:o + 4 * n] == _bytes(vl.index[0, :n]), i
        assert data[o + 4 * n:o + 6 * n] == _bytes(vl.cls[0, :n]), i
        assert data[o + 6 * n:] == _bytes(vl.xyz[0, :n]), i
