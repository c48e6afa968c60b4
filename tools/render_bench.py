#!/usr/bin/env python
"""What a camera view of a class map costs: `render_classes` alone at four shapes, and `predict_frame` against
`predict_view` of the same camera frame on the released KITTI model.

  python tools/render_bench.py [--steps K] [--warmup W] [--repeats R] [--no-model]

One JSON line per shape: after W warm-up calls, K render calls are captured into one CUDA graph and R replays are
timed with CUDA events (the median window per call is reported, every window listed), so the figure is the kernel's
and not the host's; us_per_call_unreplayed is the plain Python call, camera set-up, argument checks and launch included:
  kitti        a seeded KITTI-like map (ground plane and boxes) of 256x256x32 at 0.2 m, 1220x370, V = 2 (stereo)
  kitti_empty  an empty map of the same grid and cameras: every ray walks to its exit, the worst case
  nyu          a seeded room (floor, walls, boxes) of NYU's 60x36x60 grid ([x][z][y]) at 0.08 m, 640x480, V = 1
  scene_map    a 512x512x32 scene map (ground plane and boxes) seen from a pose yawed by 30 degrees, 1220x370, V = 1
with rays/s and the mean voxels each ray tests (from a host count over every 8th row of the oracle's walk, which
visits the same voxels).  Then one JSON line for the released KITTI model (tf32) with ms per frame of predict_frame
and of predict_view (both views), alternated.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

KITTI_ORIGIN = (0.0, -25.6, -2.0)


def _window(fn, steps):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _street(dims, seed, n_boxes):
    """uint16 [x][y][z]: road (class 9) two voxels above the bottom, sidewalk (11) at the sides, seeded boxes of car
    (1), building (13) and vegetation (15) standing on it"""
    import numpy as np
    g = np.random.default_rng(seed)
    m = np.zeros(dims, np.uint16)
    m[:, :, 8] = 9
    m[:, : dims[1] // 4, 8] = 11
    m[:, 3 * dims[1] // 4:, 8] = 11
    for _ in range(n_boxes):
        x, y = g.integers(0, dims[0] - 20), g.integers(0, dims[1] - 12)
        sx, sy, sz = g.integers(4, 20), g.integers(4, 12), g.integers(4, dims[2] - 9)
        m[x:x + sx, y:y + sy, 9:9 + sz] = g.choice([1, 13, 15])
    return m


def _room(seed):
    """uint16 [x][z][y] of NYU's 60x36x60 grid: floor (2), four walls (1), seeded boxes (5, 8, 11)"""
    import numpy as np
    g = np.random.default_rng(seed)
    m = np.zeros((60, 36, 60), np.uint16)
    m[:, 0, :] = 2
    m[0, :, :], m[-1, :, :], m[:, :, 0], m[:, :, -1] = 1, 1, 1, 1
    for _ in range(12):
        x, y = g.integers(2, 48), g.integers(2, 48)
        m[x:x + g.integers(3, 10), 1:1 + g.integers(3, 20), y:y + g.integers(3, 10)] = g.choice([5, 8, 11])
    return m


def _shapes():
    import numpy as np
    import synthetic
    from camera_frames import NYU_K, nyu_frame
    K, Ts = synthetic.kitti_calib(1220, 370)
    E2 = np.stack([np.asarray(t, np.float64) for t in Ts[:2]])[None]
    K2 = np.stack([K, K])[None]
    nyu = nyu_frame(1, with_depth=False)
    yaw = np.deg2rad(30.0)
    pose = np.eye(4)                                  # map <- velodyne: a car at (3, -2) heading 30 degrees
    pose[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    pose[:3, 3] = (3.0, -2.0, 0.0)
    E_map = np.asarray(Ts[0], np.float64) @ np.linalg.inv(pose)
    return {
        # name: (map storage [x][y][z] or [x][z][y], axes, origin, voxel, E, K, (W, H))
        "kitti": (_street((256, 256, 32), 1, 60), "xyz", KITTI_ORIGIN, 0.2, E2, K2, (1220, 370)),
        "kitti_empty": (np.zeros((256, 256, 32), np.uint16), "xyz", KITTI_ORIGIN, 0.2, E2, K2, (1220, 370)),
        "nyu": (_room(2), "xzy", nyu["vox_origin"], 0.08, np.linalg.inv(nyu["cam_pose"]), NYU_K, (640, 480)),
        "scene_map": (_street((512, 512, 32), 3, 240), "xyz", (-51.2, -51.2, -2.0), 0.2, E_map, K, (1220, 370)),
    }


def _voxels_per_ray(cmap, axes, origin, voxel, cams, W, H):
    """mean voxels tested per ray over every 8th row: the oracle walks the same voxels as the kernel"""
    import numpy as np
    from oracle import render as ref
    G, s = ref.plane_layout(cmap.shape, axes)
    rows = np.arange(0, H, 8)
    total, n = 0, 0
    for cam in cams.reshape(-1, 12):
        v, u = np.meshgrid(rows, np.arange(W), indexing="ij")
        total += int(_walk_lengths(cmap, G, s, origin, voxel, cam, u.reshape(-1), v.reshape(-1)).sum())
        n += u.size
    return total / n


def _walk_lengths(cmap, G, s, origin, voxel, cam, u, v):
    """voxels each ray tests, estimated: 1 + the boundaries it crosses between entering the grid and its hit depth
    (the oracle's) or its exit"""
    import numpy as np
    from oracle import render as ref
    _, depth, _ = ref.render(cmap, G, s, origin, voxel, cam, u, v)
    M, o = cam[:9].reshape(3, 3), cam[9:]
    d = np.stack([u, v, np.ones_like(u)], 1).astype(np.float64) @ M.T
    lo = np.asarray(origin, np.float64)
    hi = lo + np.asarray(G) * voxel
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (lo - o) / d, (hi - o) / d
    t_in = np.maximum(np.nanmax(np.minimum(t1, t2), 1), 0.0)
    t_out = np.nanmin(np.maximum(t1, t2), 1)
    t_end = np.where(np.isfinite(depth), depth.astype(np.float64), t_out)
    span = np.clip(t_end - t_in, 0, None)
    # boundaries crossed along [t_in, t_end]: |d_a| * span / voxel per axis, rounded up
    crossed = np.ceil(np.abs(d) * span[:, None] / voxel).sum(1)
    return np.where(t_out > t_in, 1 + crossed, 0)


def bench_shape(name, spec, steps, warmup, repeats):
    import torch
    from occdepth_b200 import render
    cmap_np, axes, origin, voxel, E, K, (W, H) = spec
    cmap = torch.from_numpy(cmap_np).cuda()
    view = render.render_classes(cmap, E, K, (W, H), origin, voxel, axes=axes)
    fn = lambda: render.render_classes(cmap, E, K, (W, H), origin, voxel, axes=axes, out=view)    # noqa: E731
    for _ in range(warmup):
        fn()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            fn()
    graph.replay()
    windows = [_window(graph.replay, 1) / steps for _ in range(repeats)]
    host = _window(fn, steps)
    ms = statistics.median(windows)
    B, V = view.classes.shape[:2]
    rays = B * V * H * W
    hit = float((view.index >= 0).float().mean())
    cams = render.cameras(E, K, B)
    vpr = _voxels_per_ray(cmap_np, axes, origin, voxel, cams, W, H)
    res = dict(shape=name, map=list(cmap_np.shape), axes=axes, image=[W, H], cameras=B * V, rays=rays,
               hit_fraction=round(hit, 4), voxels_per_ray_est=round(vpr, 1), us_per_call=round(ms * 1e3, 2),
               windows_us=[round(w * 1e3, 2) for w in windows], us_per_call_unreplayed=round(host * 1e3, 2),
               grays_per_s=round(rays / (ms * 1e-3) / 1e9, 3))
    del cmap, view, graph
    torch.cuda.empty_cache()
    return res


def bench_model(steps, warmup, repeats):
    import torch
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry
    name = "kitti_b3_f32_flospdepth_2080ti"
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    H, W = 370, 1220
    f = dict(kitti_frame(2, H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
    routes = {"predict_frame": lambda: m.predict_frame(f),
              "predict_view": lambda: m.predict_view(f, views=(0, 1))}
    windows = {k: [] for k in routes}
    with torch.no_grad():
        for _ in range(repeats):
            for k, fn in routes.items():
                for _ in range(max(warmup, 1)):
                    fn()
                windows[k].append(_window(fn, steps))
    med = {k: round(statistics.median(v), 4) for k, v in windows.items()}
    return dict(model=name, precision="tf32", image=[W, H], views=2, ms=med,
                windows={k: [round(x, 4) for x in v] for k, v in windows.items()},
                view_minus_predict_ms=round(med["predict_view"] - med["predict_frame"], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("render_bench: needs a CUDA device")
    import shipped_configs as sc
    card, power = sc.card()
    for name, spec in _shapes().items():
        print(json.dumps(dict(bench_shape(name, spec, a.steps, a.warmup, a.repeats), card=card, power_limit=power)),
              flush=True)
    if not a.no_model:
        print(json.dumps(dict(bench_model(max(a.steps // 20, 5), 3, a.repeats), card=card, power_limit=power)),
              flush=True)


if __name__ == "__main__":
    main()
