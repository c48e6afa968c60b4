#!/usr/bin/env python
"""What fusing a frame into a scene map costs: `SceneMap.integrate` alone at three shapes, and `predict_frame` against
`fuse_frames` of the same camera frame on the released KITTI model.

  python tools/scene_map_bench.py [--steps K] [--warmup W] [--repeats R] [--no-model]

One JSON line per shape: after W warm-up calls, K integrate calls are captured into one CUDA graph and R replays are
timed with CUDA events (the median window per call is reported, every window listed), so the figure is the kernel's
and not the host's; ms_per_call_unreplayed is the plain Python call, argument checks and launch included:
  kitti_a   C = 20, a 256x256x32 frame ([x][y][z], every voxel inside the FOV mask) into a 256x256x32 map, identity
  kitti_b   the same frame into a 512x512x32 map at a 30 degree yaw
  nyu       C = 12, a 60x36x60 frame ([x][z][y], no mask) into a 60x60x36 map, identity
with the algorithmic bytes: per observed voxel 2C (float16 probabilities) + 8C (fp32 accumulator read and write) + 8
(count read and write) + 1 (FOV byte, with a mask).  A box voxel whose centre falls outside the frame grid reads and
writes nothing.  The rate is those bytes over the kernel time, and its share of the H100 SXM's 3.35 TB/s data-sheet
bandwidth.  The probabilities are seeded softmax values; a repeated integrate keeps adding to the same map, which
does not change the work.  Then one JSON line for the released KITTI model (tf32) with ms per frame of
predict_frame(probabilities=True) and of fuse_frames into a map of the output grid's geometry, alternated.  The card's
name and power limit are read in the same run.
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

HBM_BYTES_PER_S = 3.35e12


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


def _probs(C, storage, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((C,) + storage, generator=g, device="cuda") * 2
    return torch.softmax(x, 0).half().contiguous()


def _rigid(yaw):
    import numpy as np
    T = np.eye(4)
    T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    return T


SHAPES = {
    # name: (C, storage, axes, grid origin, grid voxel, mask, map dims, map voxel, map origin, yaw)
    "kitti_a": (20, (256, 256, 32), "xyz", (0.0, -25.6, -2.0), 0.2, True, (256, 256, 32), 0.2, (0.0, -25.6, -2.0), 0.0),
    "kitti_b": (20, (256, 256, 32), "xyz", (0.0, -25.6, -2.0), 0.2, True, (512, 512, 32), 0.2, (-51.2, -51.2, -2.0),
                30.0),
    "nyu": (12, (60, 36, 60), "xzy", (-2.0, 0.5, -0.1), 0.08, False, (60, 60, 36), 0.08, (-2.0, 0.5, -0.1), 0.0),
}


def bench_shape(name, steps, warmup, repeats):
    import numpy as np
    import torch
    from occdepth_b200.fusion import SceneMap
    C, storage, axes, g, gv, with_mask, dims, voxel, origin, yaw = SHAPES[name]
    probs = _probs(C, storage, 1)
    mask = torch.ones(storage, dtype=torch.bool, device="cuda") if with_mask else None
    T = _rigid(np.deg2rad(yaw))
    smap = SceneMap(C, dims, voxel, origin)
    box = smap.integrate(probs, T, g, gv, axes=axes, fov_mask=mask)
    observed = int(smap.count.sum())
    fn = lambda: smap.integrate(probs, T, g, gv, axes=axes, fov_mask=mask)       # noqa: E731
    for _ in range(warmup):
        fn()
    # the K launches replayed from one CUDA graph: the window times the kernels, not the host's argument checks
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(steps):
            fn()
    graph.replay()
    windows = [_window(graph.replay, 1) / steps for _ in range(repeats)]
    host = _window(fn, steps)
    ms = statistics.median(windows)
    nbytes = observed * (10 * C + 8 + (1 if with_mask else 0))
    box_voxels = (box[1] - box[0]) * (box[3] - box[2]) * (box[5] - box[4])
    res = dict(shape=name, C=C, frame=list(storage), map=list(dims), yaw_deg=yaw, box_voxels=box_voxels,
               observed_voxels=observed, algorithmic_bytes=nbytes, ms=round(ms, 5),
               windows=[round(w, 5) for w in windows], ms_per_call_unreplayed=round(host, 5), gb_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1),
               share_of_3_35_tb_s=round(nbytes / HBM_BYTES_PER_S / (ms * 1e-3), 3))
    del smap, probs, graph
    torch.cuda.empty_cache()
    return res


def bench_model(steps, warmup, repeats):
    import numpy as np
    import torch
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry
    from occdepth_b200.fusion import SceneMap
    name = "kitti_b3_f32_flospdepth_2080ti"
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision("tf32")
    H, W = sc.KITTI_IMG
    f = dict(kitti_frame(sc.CONFIGS[name]["views"], H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
    smap = SceneMap(m.n_classes, sc.KITTI_FULL, 0.2, f["vox_origin"])
    routes = {"predict_frame_probs": lambda: m.predict_frame(f, probabilities=True),
              "fuse_frames": lambda: m.fuse_frames(smap, f, np.eye(4))}
    windows = {k: [] for k in routes}
    with torch.no_grad():
        for _ in range(repeats):
            for k, fn in routes.items():
                for _ in range(max(warmup, 1)):
                    fn()
                windows[k].append(_window(fn, steps))
    med = {k: round(statistics.median(v), 4) for k, v in windows.items()}
    return dict(model=name, precision="tf32", ms=med, windows={k: [round(x, 4) for x in v] for k, v in windows.items()},
                fuse_minus_predict_ms=round(med["fuse_frames"] - med["predict_frame_probs"], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("scene_map_bench: needs a CUDA device")
    import shipped_configs as sc
    card, power = sc.card()
    for name in SHAPES:
        print(json.dumps(dict(bench_shape(name, a.steps, a.warmup, a.repeats), card=card, power_limit=power)),
              flush=True)
    if not a.no_model:
        print(json.dumps(dict(bench_model(max(a.steps // 20, 5), 3, a.repeats), card=card, power_limit=power)),
              flush=True)


if __name__ == "__main__":
    main()
