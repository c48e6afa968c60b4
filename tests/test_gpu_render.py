"""Camera views on the device (occd_render_classes, render.render_classes, SceneMap.render, OccDepth.predict_view)
against the numpy restatement in oracle/render.py bit for bit, and across the Python routes."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import render
from occdepth_b200.fusion import SceneMap
from oracle import render as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402
from test_render_host import intrinsics, look, random_map  # noqa: E402


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _check_rows(cmap, axes, origin, voxel, cams, view, rows, **kw):
    """every (b, v) image of `view` on rows `rows` against the oracle, bit for bit; returns the hit count"""
    maps = cmap.cpu().numpy()
    hits = 0
    B, V, H, W = view.classes.shape
    got = [x.cpu().numpy() for x in view]
    for b in range(B):
        G, s = ref.plane_layout(maps[b].shape, axes)
        for v in range(V):
            want = ref.render_image(maps[b], G, s, origin, voxel, cams[b, v], W, H, rows, **kw)
            for g, w in zip(got, want):
                assert g[b, v, rows].tobytes() == w.tobytes(), (b, v)
            hits += int((want[2] >= 0).sum())
    return hits


def _random_case(axes, seed):
    storage = (40, 36, 12) if axes == "xyz" else (40, 12, 36)
    G, _ = ref.plane_layout(storage, axes)
    voxel, origin = 0.2, np.array([-1.0, -3.6, -1.2])
    maps = np.stack([random_map(storage, 0.08, seed + b) for b in range(2)])
    centre = origin + np.asarray(G) * voxel / 2
    # per map: a camera outside looking in, and one inside the grid
    E = np.stack([np.stack([look(centre - np.array([6.0, 1.0 * b, -1.5]), 0.05 * b, 0.25),
                            look(centre + np.array([0.2, 0.3, 0.1]), 2.0 + b, 0.1)]) for b in range(2)])
    K = intrinsics(80.0, 96, 64)
    return torch.from_numpy(maps).cuda(), E, K, origin, voxel


@pytest.mark.parametrize("axes", ["xyz", "xzy"])
def test_kernel_matches_the_oracle(axes):
    cmap, E, K, origin, voxel = _random_case(axes, 1)
    cams = render.cameras(E, K, B=2)
    for kw in (dict(), dict(near=1.0, far=6.0), dict(empty=255, ignore=0)):
        view = render.render_classes(cmap, E, K, (96, 64), origin, voxel, axes=axes, **kw)
        assert view.classes.shape == (2, 2, 64, 96)
        hits = _check_rows(cmap, axes, origin, voxel, cams, view, np.arange(64), **kw)
        assert 0 < hits < 2 * 2 * 64 * 96


def test_every_output_subset_gives_the_same_bytes_and_is_deterministic():
    cmap, E, K, origin, voxel = _random_case("xyz", 2)
    full = render.render_classes(cmap, E, K, (96, 64), origin, voxel)
    again = render.render_classes(cmap, E, K, (96, 64), origin, voxel)
    assert all(_same(a, b) for a, b in zip(full, again))
    for mask in range(1, 8):
        out = render.View(*(torch.full_like(x, 77) if mask >> i & 1 else None for i, x in enumerate(full)))
        got = render.render_classes(cmap, E, K, (96, 64), origin, voxel, out=out)
        for i in range(3):
            if mask >> i & 1:
                assert got[i] is out[i] and _same(got[i], full[i]), (mask, i)


def test_cuda_graph_capture():
    cmap, E, K, origin, voxel = _random_case("xzy", 3)
    want = render.render_classes(cmap, E, K, (96, 64), origin, voxel, axes="xzy")
    out = render.View(*(torch.zeros_like(x) for x in want))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        render.render_classes(cmap, E, K, (96, 64), origin, voxel, axes="xzy", out=out)      # warm-up
    torch.cuda.current_stream().wait_stream(s)
    for x in out:
        x.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        render.render_classes(cmap, E, K, (96, 64), origin, voxel, axes="xzy", out=out)
    g.replay()
    torch.cuda.synchronize()
    assert all(_same(a, b) for a, b in zip(out, want))


# ---- models ----------------------------------------------------------------------------------------------------------
def _n_plans(m):
    return len(m._plans()) + len(m._class_plans())


def test_kitti_stereo_frame_view():
    import shipped_configs as sc
    _free()
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti")
    m = m.cuda().set_precision("tf32")
    H, W = 370, 1220
    f = dict(kitti_frame(2, H, W, 4), **kitti_geometry(H, W, sc.KITTI_FULL))
    with torch.no_grad():
        y0 = m.predict_frame(f).clone()
        n0 = _n_plans(m)
        y, view = m.predict_view(f, views=(0, 1))
        assert _n_plans(m) == n0                                        # the class-map plan, under its key
        assert _same(y, y0)
        E, K = f["T_velo_2_cam"][None], f["cam_k"][None]
        want = render.render_classes(y, E, K, (W, H), f["vox_origin"], 0.2)
    assert view.classes.shape == (1, 2, H, W)
    assert all(_same(a, b) for a, b in zip(view, want))
    rows = np.arange(0, H, 16)
    hits = _check_rows(y, "xyz", f["vox_origin"], 0.2, render.cameras(E, K), view, rows)
    print("kitti: %d of %d checked rays hit a voxel" % (hits, 2 * len(rows) * W))
    assert hits > 0
    # a batch of two frames: one launch, the same bytes as each frame alone
    f2 = dict(kitti_frame(2, H, W, 5, shift=0.4), **kitti_geometry(H, W, sc.KITTI_FULL))
    with torch.no_grad():
        yb, vb = m.predict_view([f, f2], views=(1,))
        y2, v2 = m.predict_view(f2, views=(1,))
    assert _same(vb.classes[0], view.classes[0, 1:]) and _same(vb.depth[1], v2.depth[0])
    assert _same(vb.index[1], v2.index[0]) and _same(yb[1], y2[0])
    del m
    _free()


def test_nyu_frame_view():
    import shipped_configs as sc
    _free()
    m, _, _ = sc.make_case("nyu_b4_f100_2080ti")
    m = m.cuda().set_precision("tf32")
    f = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
    H, W = sc.NYU_IMG
    with torch.no_grad():
        y, view = m.predict_view(f, views=(0, 1))                       # the camera and the virtual right view
        y0 = m.predict_frame(f)
        fi = m._frame_inputs(f, torch.device("cuda"))
        E = np.stack([p[0] for p in fi["poses"]])[None]
        K = np.stack([p[1] for p in fi["poses"]])[None]
        want = render.render_classes(y0, E, K, (W, H), f["vox_origin"], 0.08, axes="xzy")
    assert _same(y, y0) and view.classes.shape == (1, 2, H, W)
    assert all(_same(a, b) for a, b in zip(view, want))
    hits = _check_rows(y, "xzy", f["vox_origin"], 0.08, render.cameras(E, K), view, np.arange(0, H, 8))
    assert hits > 0
    del m
    _free()


def test_scene_map_render_after_fuse_frames():
    import shipped_configs as sc
    _free()
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=(96, 320), full=(64, 64, 16))
    m = m.cuda().set_precision("tf32")
    H, W = 96, 320
    frames = [dict(kitti_frame(2, H, W, 1 + i, shift=0.3 * i), **kitti_geometry(H, W, (64, 64, 16))) for i in range(2)]
    with torch.no_grad():
        smap = SceneMap(m.n_classes, (80, 80, 16), 0.2, (-1.0, -8.0, -2.0))
        m.fuse_frames(smap, frames, [np.eye(4)] * 2)
        E, K = frames[0]["T_velo_2_cam"][0], frames[0]["cam_k"][0]          # map frame = velodyne frame
        got = smap.render(E, K, (W, H), far=40.0)
        want = render.render_classes(smap.classes(), E, K, (W, H), smap.origin, smap.voxel, ignore=255, far=40.0)
    assert got.classes.shape == (1, 1, H, W)
    assert all(_same(a, b) for a, b in zip(got, want))
    assert bool((got.index >= 0).any()) and not bool((got.classes == 255).any())
    del m
    _free()
