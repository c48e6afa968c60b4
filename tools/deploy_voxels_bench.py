#!/usr/bin/env python
"""Occupied-voxel lists from model files against the dense map: ms per frame and bytes read back per frame of
`occd_model_run_frames` plus the class map's read-back, and of the same run plus `occd_model_list_voxels` plus the
read-back of the counts, the histogram and the written rows -- per configuration (the released KITTI and NYU models
and the EfficientNet-B7 FlospDepth one) in both precisions, at the shipped shapes.

  python tools/deploy_voxels_bench.py [--steps K] [--warmup W] [--windows R] [--precision tf32|bf16] [names...]

Both routes run one frame per step on the current stream and end each step with the host holding the result (a
pinned buffer): the map route copies the whole uint16 map; the list route copies the counts and histogram, waits for
them, then copies the written rows (int32 index, uint16 class, float32 x, y, z).  Each window is K steps after W
warm-up steps, timed with CUDA events; the routes alternate window by window (R windows each, medians reported, every
window listed).  A KITTI frame keeps its calibration, so the indices and the FOV mask are not recomputed.  The lists
are checked against OccDepth.predict_voxels of the same frame.  The card's name and power limit are read in the same
run.  Model files go to a temporary directory.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

CONFIGS = ("kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti", "kitti_b7_f64_flospdepth_a100")


def _window(fn, steps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    import shipped_configs as sc
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("deploy_voxels_bench.py measures on a CUDA (sm_90a) device; none is visible")
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from occdepth_b200 import deploy
    from occdepth_b200.voxels import HIST_BINS
    gpu, power = sc.card()
    tmp = tempfile.mkdtemp(prefix="occd_deploy_voxels_bench_")
    for name in a.names:
        m, _, _ = sc.make_case(name)
        m = m.cuda()
        nyu = sc.CONFIGS[name]["dataset"] == "NYU"
        if nyu:
            frame = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
        else:
            H, W = sc.KITTI_IMG
            frame = dict(kitti_frame(sc.CONFIGS[name]["views"], H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
        frame["img"] = torch.from_numpy(frame["img"]).cuda()      # device images, as a decoder hands them over
        if nyu:
            frame["depth"] = torch.from_numpy(frame["depth"]).cuda()
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            path = os.path.join(tmp, "%s_%s.occd" % (name, prec))
            with torch.no_grad():
                deploy.export(m, path, frame)
                want = m.predict_voxels(frame)
                torch.cuda.synchronize()
                cm = deploy.LoadedModel(path)
                g = cm.geom
                out = torch.empty(1, g.X, g.Y, g.Z, dtype=torch.uint16, device="cuda")
                h_map = torch.empty(out.shape, dtype=torch.uint16, pin_memory=True)
                cm.run_frames([frame], out=out)
                vl = cm.list_voxels()
                N = g.X * g.Y * g.Z
                h_head = torch.empty(2 + HIST_BINS, dtype=torch.int32, pin_memory=True)
                h_index = torch.empty(N, dtype=torch.int32, pin_memory=True)
                h_cls = torch.empty(N, dtype=torch.uint16, pin_memory=True)
                h_xyz = torch.empty(N, 3, dtype=torch.float32, pin_memory=True)
                read = {"map": 0, "voxels": 0}

                def run_map():
                    cm.run_frames([frame], out=out)
                    h_map.copy_(out, non_blocking=True)
                    torch.cuda.current_stream().synchronize()
                    read["map"] = h_map.numel() * 2

                def run_voxels():
                    cm.run_frames([frame], out=out)
                    cm.list_voxels(out=vl)
                    h_head[:2].copy_(vl.count[0], non_blocking=True)
                    h_head[2:].copy_(vl.hist[0], non_blocking=True)
                    torch.cuda.current_stream().synchronize()
                    n = min(int(h_head[0]) + int(h_head[1]), vl.capacity)
                    h_index[:n].copy_(vl.index[0, :n], non_blocking=True)
                    h_cls[:n].copy_(vl.cls[0, :n], non_blocking=True)
                    h_xyz[:n].copy_(vl.xyz[0, :n], non_blocking=True)
                    torch.cuda.current_stream().synchronize()
                    read["voxels"] = h_head.numel() * 4 + n * (4 + 2 + 12)
                routes = {"map": run_map, "voxels": run_voxels}
                for fn in routes.values():
                    for _ in range(a.warmup):
                        fn()
                ms = {k: [] for k in routes}
                for _ in range(a.windows):
                    for k, fn in routes.items():
                        ms[k].append(_window(fn, a.steps))
                n = int(want.counts()[0].sum())
                same = (vl.counts().tolist() == want.counts().tolist() and
                        all(torch.equal(getattr(vl, k)[0, :n].view(torch.uint8), getattr(want, k)[0, :n].view(torch.uint8))
                            for k in ("index", "cls", "xyz")) and torch.equal(vl.hist, want.hist))
            cm.close()
            os.remove(path)
            print(json.dumps(dict(
                config=name, precision=prec,
                run_map_ms=round(statistics.median(ms["map"]), 3),
                run_list_voxels_ms=round(statistics.median(ms["voxels"]), 3),
                run_map_windows_ms=[round(t, 3) for t in ms["map"]],
                run_list_voxels_windows_ms=[round(t, 3) for t in ms["voxels"]],
                map_bytes_read_per_frame=read["map"], list_bytes_read_per_frame=read["voxels"],
                occupied=[int(v) for v in np.asarray(vl.counts()[0])], lists_equal=bool(same),
                steps=a.steps, warmup=a.warmup, gpu=gpu, power_limit=power)), flush=True)
        del m
        torch.cuda.empty_cache()
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
