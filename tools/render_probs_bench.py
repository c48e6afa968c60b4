#!/usr/bin/env python
"""What a soft camera view costs: `render_probs` alone at four shapes, the hard render of the same map beside the
one-hot field, and `predict_view(soft=True)` against `predict_view` on the released KITTI model.

  python tools/render_probs_bench.py [--steps K] [--warmup W] [--repeats R] [--no-model]

One JSON line per shape: after W warm-up calls, K calls are captured into one CUDA graph and R replays are timed with
CUDA events (the median window per call is reported, every window listed), so the figure is the kernel's:
  kitti_soft     a seeded KITTI-like probability field, 256x256x32 at 0.2 m, C = 20: free space (p(empty) == 1
                 exactly), soft surfaces a ray crosses partly, confident ones; two 1220x370 cameras; default t_min
  kitti_soft_t0  the same with min_transmittance = 0: every ray walks until T is exactly 0 or it leaves the grid
  kitti_onehot   the one-hot field of the same arg-max map, and kitti_hard: render_classes of that map
  nyu            NYU's 60x36x60 grid ([x][z][y]) at 0.08 m, C = 12, 640x480, V = 1
  scene_map      a 512x512x32 map (C = 20) from a pose yawed by 30 degrees, 1220x370, V = 1
Per ray, counted on the host over every 8th row by the oracle's walk with the kernel's skip and stop rules: voxels
visited, voxels read (not skipped: every channel loaded) and bytes gathered (2 per float16 channel read, 2 for the
empty channel of a skipped voxel); gather_gb_per_s is those bytes over the kernel time.  Then one JSON line for the
released KITTI model (tf32): ms per frame of predict_view and predict_view(soft=True), alternated.  The card's name
and power limit are read in the same run.
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

from render_bench import KITTI_ORIGIN, _room, _street, _window  # noqa: E402


def _soften(cmap, seed, Cn):
    """float16 [C, ...] from a class map: empty voxels certainly free (p(empty) == 1 exactly); an occupied voxel's
    p(empty) drawn so that a third of the surfaces are soft (0.3 .. 0.8) and the rest confident (0 .. 0.05), its
    class holding 0.8 of the occupied mass and every other class an equal share; half the free voxels in front of a
    surface (along the contiguous axis) hold a faint haze, p(empty) 0.9 .. 1, that rays cross"""
    import numpy as np
    g = np.random.default_rng(seed)
    occ = cmap != 0
    pe = np.where(g.random(cmap.shape) < 1 / 3, g.uniform(0.3, 0.8, cmap.shape), g.uniform(0.0, 0.05, cmap.shape))
    haze = np.zeros(cmap.shape, bool)
    haze[..., :-1] = occ[..., 1:]
    pe = np.where(occ, pe, np.where(haze & (g.random(cmap.shape) < 0.5), g.uniform(0.9, 1.0, cmap.shape), 1.0))
    k = np.clip(cmap.astype(np.int64), 1, Cn - 1)
    p = np.empty((Cn,) + cmap.shape, np.float16)
    p[0] = pe
    share = (1 - pe) * 0.2 / max(Cn - 2, 1)
    for c in range(1, Cn):
        p[c] = np.where(k == c, (1 - pe) * 0.8, share)
    return p


def _one_hot(cmap, Cn):
    import numpy as np
    p = np.zeros((Cn,) + cmap.shape, np.float16)
    for c in range(Cn):
        p[c][cmap == c] = 1
    return p


def _shapes():
    import numpy as np
    import synthetic
    from camera_frames import NYU_K, nyu_frame
    K, Ts = synthetic.kitti_calib(1220, 370)
    E2 = np.stack([np.asarray(t, np.float64) for t in Ts[:2]])[None]
    K2 = np.stack([K, K])[None]
    nyu = nyu_frame(1, with_depth=False)
    yaw = np.deg2rad(30.0)
    pose = np.eye(4)
    pose[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    pose[:3, 3] = (3.0, -2.0, 0.0)
    E_map = np.asarray(Ts[0], np.float64) @ np.linalg.inv(pose)
    street = _street((256, 256, 32), 1, 60)
    soft = _soften(street, 1, 20)
    room = _room(2)
    room[room >= 12] = 11
    big = _street((512, 512, 32), 3, 240)
    return {
        # name: (probs [C, storage], class map for the hard twin or None, axes, origin, voxel, E, K, (W, H), t_min)
        "kitti_soft": (soft, None, "xyz", KITTI_ORIGIN, 0.2, E2, K2, (1220, 370), 1e-4),
        "kitti_soft_t0": (soft, None, "xyz", KITTI_ORIGIN, 0.2, E2, K2, (1220, 370), 0.0),
        "kitti_onehot": (_one_hot(street, 20), street, "xyz", KITTI_ORIGIN, 0.2, E2, K2, (1220, 370), 1e-4),
        "nyu": (_soften(room, 2, 12), None, "xzy", nyu["vox_origin"], 0.08, np.linalg.inv(nyu["cam_pose"]),
                NYU_K, (640, 480), 1e-4),
        "scene_map": (_soften(big, 3, 20), None, "xyz", (-51.2, -51.2, -2.0), 0.2, E_map, K, (1220, 370),
                      1e-4),
    }


def _gather_stats(probs, axes, origin, voxel, cams, W, H, t_min):
    """per ray over every 8th row: voxels visited, voxels read in full, bytes gathered (the kernel's rules)"""
    import numpy as np
    from oracle import render_probs as ref
    Cn = probs.shape[0]
    G, s = ref.plane_layout(probs.shape[1:], axes)
    P = probs.reshape(Cn, -1)
    rows = np.arange(0, H, 8)
    visited = read = rays = 0
    for cam in cams.reshape(-1, 12):
        v, u = np.meshgrid(rows, np.arange(W), indexing="ij")
        T = np.ones(u.size, np.float32)
        cnt = np.zeros(2, np.int64)

        def visit(act, off, t):
            e = P[0, off].astype(np.float32)
            full = e != np.float32(1)
            cnt[0] += act.size
            cnt[1] += int(full.sum())
            a = act[full]
            T[a] = T[a] * e[full]
            stop = np.zeros(act.size, bool)
            stop[full] = T[a] <= np.float32(t_min)
            return stop

        ref.walk(G, s, origin, voxel, cam, u.reshape(-1), v.reshape(-1), visit)
        visited += int(cnt[0])
        read += int(cnt[1])
        rays += u.size
    return visited / rays, read / rays, (2 * visited + 2 * (Cn - 1) * read) / rays


def _graph_time(fn, steps, warmup, repeats):
    import torch
    for _ in range(warmup):
        fn()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            fn()
    graph.replay()
    windows = [_window(graph.replay, 1) / steps for _ in range(repeats)]
    del graph
    return statistics.median(windows), windows


def bench_shape(name, spec, steps, warmup, repeats):
    import torch
    from occdepth_b200 import render
    probs_np, cmap_np, axes, origin, voxel, E, K, (W, H), t_min = spec
    probs = torch.from_numpy(probs_np).cuda()
    view = render.render_probs(probs, E, K, (W, H), origin, voxel, axes=axes, min_transmittance=t_min)
    fn = lambda: render.render_probs(probs, E, K, (W, H), origin, voxel, axes=axes,   # noqa: E731
                                     min_transmittance=t_min, out=view)
    ms, windows = _graph_time(fn, steps, warmup, repeats)
    B, V = view.classes.shape[:2]
    rays = B * V * H * W
    cams = render.cameras(E, K, B)
    vpr, rpr, bpr = _gather_stats(probs_np, axes, origin, voxel, cams, W, H, t_min)
    res = dict(shape=name, map=list(probs_np.shape), axes=axes, image=[W, H], cameras=B * V, rays=rays,
               t_min=t_min, mean_opacity=round(float(view.opacity.mean()), 4), voxels_visited_per_ray=round(vpr, 1),
               voxels_read_per_ray=round(rpr, 1), bytes_gathered_per_ray=round(bpr, 1),
               us_per_call=round(ms * 1e3, 2), windows_us=[round(w * 1e3, 2) for w in windows],
               grays_per_s=round(rays / (ms * 1e-3) / 1e9, 3),
               gather_gb_per_s=round(bpr * rays / (ms * 1e-3) / 1e9, 1))
    out = [res]
    if cmap_np is not None:                              # the hard render of the same map: soft's price
        cmap = torch.from_numpy(cmap_np).cuda()
        hv = render.render_classes(cmap, E, K, (W, H), origin, voxel, axes=axes)
        assert torch.equal(hv.classes, view.classes) and torch.equal(hv.depth, view.depth)
        hfn = lambda: render.render_classes(cmap, E, K, (W, H), origin, voxel, axes=axes, out=hv)  # noqa: E731
        hms, hw = _graph_time(hfn, steps, warmup, repeats)
        out.append(dict(shape=name.replace("onehot", "hard"), map=list(cmap_np.shape), image=[W, H],
                        cameras=B * V, us_per_call=round(hms * 1e3, 2), windows_us=[round(w * 1e3, 2) for w in hw],
                        soft_over_hard=round(ms / hms, 2)))
        del cmap, hv
    del probs, view
    torch.cuda.empty_cache()
    return out


def bench_model(steps, warmup, repeats):
    import torch
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry
    name = "kitti_b3_f32_flospdepth_2080ti"
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    H, W = 370, 1220
    f = dict(kitti_frame(2, H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
    routes = {"predict_view": lambda: m.predict_view(f, views=(0, 1)),
              "predict_view_soft": lambda: m.predict_view(f, views=(0, 1), soft=True)}
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
                soft_minus_hard_ms=round(med["predict_view_soft"] - med["predict_view"], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("render_probs_bench: needs a CUDA device")
    import shipped_configs as sc
    card, power = sc.card()
    for name, spec in _shapes().items():
        for res in bench_shape(name, spec, a.steps, a.warmup, a.repeats):
            print(json.dumps(dict(res, card=card, power_limit=power)), flush=True)
    if not a.no_model:
        print(json.dumps(dict(bench_model(max(a.steps // 10, 5), 3, a.repeats), card=card, power_limit=power)),
              flush=True)


if __name__ == "__main__":
    main()
