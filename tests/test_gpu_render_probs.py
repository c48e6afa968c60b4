"""Soft camera views on the device (occd_render_probs, render.render_probs, SceneMap.render_probs,
OccDepth.predict_view(soft=True)) against the numpy restatement in oracle/render_probs.py bit for bit, against the
hard render on one-hot fields, and across the Python routes."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import render
from occdepth_b200.fusion import SceneMap
from oracle import render_probs as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402
from test_render_host import intrinsics, look, random_map  # noqa: E402
from test_render_probs_host import canon, soft_field  # noqa: E402


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _check_rows(probs, axes, origin, voxel, cams, view, rows, class_map=None, **kw):
    """every (b, v) image of SoftView `view` on rows `rows` against the oracle, bit for bit; returns the mean opacity"""
    P = probs.cpu().numpy()
    cm = None if class_map is None else class_map.cpu().numpy()
    B, V, H, W = view.classes.shape
    got = [x.cpu().numpy() for x in view]
    opa = []
    for b in range(B):
        G, s = ref.plane_layout(P.shape[2:], axes)
        for v in range(V):
            want = ref.render_probs_image(P[b], G, s, origin, voxel, cams[b, v], W, H, rows,
                                          class_map=None if cm is None else cm[b], **kw)
            for name, g, w in zip(("cls", "depth", "opacity"), got[:3], want[:3]):
                assert canon(g[b, v, rows]) == canon(w), (name, b, v)
            assert canon(got[3][b, v][:, rows]) == canon(want[3]), ("probs", b, v)
            opa.append(float(want[2].mean()))
    return float(np.mean(opa))


def _random_case(axes, seed, Cn):
    storage = (40, 36, 12) if axes == "xyz" else (40, 12, 36)
    G, _ = ref.plane_layout(storage, axes)
    voxel, origin = 0.2, np.array([-1.0, -3.6, -1.2])
    fields = [soft_field(storage, Cn, seed + b, surface=0.03, free=0.85) for b in range(2)]
    probs = np.stack([f[0] for f in fields])
    cmap = np.stack([f[1] for f in fields])
    centre = origin + np.asarray(G) * voxel / 2
    E = np.stack([np.stack([look(centre - np.array([6.0, 1.0 * b, -1.5]), 0.05 * b, 0.25),
                            look(centre + np.array([0.2, 0.3, 0.1]), 2.0 + b, 0.1)]) for b in range(2)])
    K = intrinsics(80.0, 96, 64)
    return torch.from_numpy(probs).cuda(), torch.from_numpy(cmap).cuda(), E, K, origin, voxel


@pytest.mark.parametrize("axes,Cn", [("xyz", 20), ("xzy", 12), ("xyz", 33), ("xzy", 64), ("xyz", 3)])
def test_kernel_matches_the_oracle(axes, Cn):
    probs, cmap, E, K, origin, voxel = _random_case(axes, 1, Cn)
    cams = render.cameras(E, K, B=2)
    lut = np.random.default_rng(Cn).integers(0, 300, Cn)
    for kw in (dict(), dict(near=1.0, far=6.0, min_transmittance=0.0),
               dict(class_map=cmap, ignore=255, inv_map=lut, min_transmittance=0.05)):
        view = render.render_probs(probs, E, K, (96, 64), origin, voxel, axes=axes, **kw)
        assert view.classes.shape == (2, 2, 64, 96) and view.probs.shape == (2, 2, Cn, 64, 96)
        okw = dict(near=kw.get("near", 0.0), far=kw.get("far", np.inf), t_min=kw.get("min_transmittance", 1e-4),
                   lut=kw.get("inv_map"), ignore=kw.get("ignore", 255))
        mean_opacity = _check_rows(probs, axes, origin, voxel, cams, view, np.arange(64), kw.get("class_map"), **okw)
        assert 0.0 < mean_opacity < 1.0


def test_every_output_subset_gives_the_same_bytes_and_is_deterministic():
    probs, cmap, E, K, origin, voxel = _random_case("xyz", 2, 20)
    go = lambda **kw: render.render_probs(probs, E, K, (96, 64), origin, voxel, class_map=cmap, **kw)  # noqa: E731
    full = go()
    again = go()
    assert all(_same(a, b) for a, b in zip(full, again))
    for mask in range(1, 16):
        out = render.SoftView(*(torch.full_like(x, 77) if mask >> i & 1 else None for i, x in enumerate(full)))
        got = go(out=out)
        for i in range(4):
            if mask >> i & 1:
                assert got[i] is out[i] and _same(got[i], full[i]), (mask, i)


def test_cuda_graph_capture():
    probs, cmap, E, K, origin, voxel = _random_case("xzy", 3, 17)
    go = lambda out=None: render.render_probs(probs, E, K, (96, 64), origin, voxel, axes="xzy",  # noqa: E731
                                              min_transmittance=0.0, out=out)
    want = go()
    out = render.SoftView(*(torch.zeros_like(x) for x in want))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        go(out)                                                                          # warm-up
    torch.cuda.current_stream().wait_stream(s)
    for x in out:
        x.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        go(out)
    g.replay()
    torch.cuda.synchronize()
    assert all(_same(a, b) for a, b in zip(out, want))


@pytest.mark.parametrize("axes", ["xyz", "xzy"])
def test_one_hot_render_is_the_hard_render(axes):
    storage = (40, 36, 12) if axes == "xyz" else (40, 12, 36)
    Cn = 20
    maps = np.stack([random_map(storage, 0.08, 5 + b, classes=Cn) for b in range(2)])
    probs = np.zeros((2, Cn) + storage, np.float16)
    for c in range(Cn):
        probs[:, c][maps == c] = 1
    cmap = torch.from_numpy(maps).cuda()
    _, _, E, K, origin, voxel = _random_case(axes, 1, 3)
    soft = render.render_probs(torch.from_numpy(probs).cuda(), E, K, (96, 64), origin, voxel, axes=axes,
                               class_map=cmap)
    hard = render.render_classes(cmap, E, K, (96, 64), origin, voxel, axes=axes)
    assert _same(soft.classes, hard.classes) and _same(soft.depth, hard.depth)
    assert torch.equal(soft.opacity, (hard.index >= 0).float())
    hit = hard.index >= 0
    assert bool(hit.any()) and not bool(hit.all())


def test_frame_views_of_frames_with_their_own_grids():
    """predict_view's per-frame route (NYU frames with their own vox_origin): each frame rendered alone into its
    slice, the same bytes as separate calls, for both renders"""
    from occdepth_b200.models.OccDepth import OccDepth
    probs, cmap, E, K, origin, voxel = _random_case("xzy", 4, 12)
    reqs = [dict(E=E[b:b + 1], K=K, size=(96, 64), grid_origin=origin + 0.1 * b, grid_voxel=voxel, axes="xzy")
            for b in range(2)]
    for fn, x, kw in ((render.render_probs, probs, dict(min_transmittance=0.0)), (render.render_classes, cmap, {})):
        got = OccDepth._frame_views(fn, x, reqs, **kw)
        for b in range(2):
            want = fn(x[b:b + 1], **reqs[b], **kw)
            assert all(_same(g[b:b + 1], w) for g, w in zip(got, want)), (fn.__name__, b)


# ---- models ----------------------------------------------------------------------------------------------------------
def _n_plans(m):
    return len(m._plans()) + len(m._class_plans())


def test_kitti_stereo_frame_soft_view():
    import shipped_configs as sc
    _free()
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti")
    m = m.cuda().set_precision("tf32")
    H, W = 370, 1220
    f = dict(kitti_frame(2, H, W, 4), **kitti_geometry(H, W, sc.KITTI_FULL))
    with torch.no_grad():
        y0, p0 = (x.clone() for x in m.predict_frame(f, probabilities=True))
        n0 = _n_plans(m)
        y, p, view = m.predict_view(f, views=(0, 1), soft=True)
        assert _n_plans(m) == n0                                        # the probabilities plan, under its key
        assert _same(y, y0) and _same(p, p0)
        E, K = f["T_velo_2_cam"][None], f["cam_k"][None]
        want = render.render_probs(p, E, K, (W, H), f["vox_origin"], 0.2)
    assert view.classes.shape == (1, 2, H, W) and view.probs.shape == (1, 2, m.n_classes, H, W)
    assert all(_same(a, b) for a, b in zip(view, want))
    rows = np.arange(0, H, 37)
    opa = _check_rows(p, "xyz", f["vox_origin"], 0.2, render.cameras(E, K), view, rows)
    print("kitti: mean opacity %.3f over the checked rows" % opa)
    # a batch of two frames: one launch, the same bytes as each frame alone
    f2 = dict(kitti_frame(2, H, W, 5, shift=0.4), **kitti_geometry(H, W, sc.KITTI_FULL))
    with torch.no_grad():
        yb, pb, vb = m.predict_view([f, f2], views=(1,), soft=True)
        y2, p2, v2 = m.predict_view(f2, views=(1,), soft=True)
    for i in range(4):
        assert _same(vb[i][0], view[i][0, 1:]) and _same(vb[i][1], v2[i][0]), i
    assert _same(yb[1], y2[0]) and _same(pb[1], p2[0])
    del m
    _free()


def test_nyu_frame_soft_view():
    import shipped_configs as sc
    _free()
    m, _, _ = sc.make_case("nyu_b4_f100_2080ti")
    m = m.cuda().set_precision("tf32")
    f = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
    H, W = sc.NYU_IMG
    with torch.no_grad():
        y, p, view = m.predict_view(f, views=(0, 1), soft=True)       # the camera and the virtual right view
        y0, p0 = m.predict_frame(f, probabilities=True)
        fi = m._frame_inputs(f, torch.device("cuda"))
        E = np.stack([q[0] for q in fi["poses"]])[None]
        K = np.stack([q[1] for q in fi["poses"]])[None]
        want = render.render_probs(p0, E, K, (W, H), f["vox_origin"], 0.08, axes="xzy")
    assert _same(y, y0) and _same(p, p0) and view.classes.shape == (1, 2, H, W)
    assert all(_same(a, b) for a, b in zip(view, want))
    _check_rows(p, "xzy", f["vox_origin"], 0.08, render.cameras(E, K), view, np.arange(0, H, 24))
    del m
    _free()


def test_scene_map_render_probs_after_fuse_frames():
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
        got = smap.render_probs(E, K, (W, H), far=40.0)
        cmap, probs = smap.classes(probabilities=True)
        want = render.render_probs(probs, E, K, (W, H), smap.origin, smap.voxel, class_map=cmap, ignore=255,
                                   far=40.0)
        # unobserved voxels contribute nothing: the same view with their probabilities overwritten
        unobserved = (smap.count == 0)
        assert bool(unobserved.any()) and bool((~unobserved).any())
        noisy = probs.clone()
        noisy[:, unobserved] = torch.tensor(0.5, dtype=torch.float16, device=noisy.device)
        masked = render.render_probs(noisy, E, K, (W, H), smap.origin, smap.voxel, class_map=cmap, ignore=255,
                                     far=40.0)
        # and without the class map they would: the same probabilities render differently
        opaque = render.render_probs(probs, E, K, (W, H), smap.origin, smap.voxel, far=40.0)
    assert got.classes.shape == (1, 1, H, W)
    assert all(_same(a, b) for a, b in zip(got, want))
    assert all(_same(a, b) for a, b in zip(masked, want))
    assert not _same(opaque.opacity, got.opacity)
    assert bool((got.opacity > 0).any())
    _check_rows(probs[None], "xyz", smap.origin, smap.voxel, render.cameras(E, K), got, np.arange(0, H, 12),
                cmap[None], far=40.0)
    del m
    _free()
