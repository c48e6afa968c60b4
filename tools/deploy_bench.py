#!/usr/bin/env python
"""Python-free route against predict_frame: ms per frame of `occd_model_run_frame` (a model file exported by
occdepth_b200.deploy, replayed by the C runtime) and of `OccDepth.predict_frame` on the same frame, per shipped
configuration at its shipped shapes.

  python tools/deploy_bench.py [--steps K] [--warmup W] [--windows R] [names...]

Both routes run on the current stream; each window is K frames after W warm-up frames, timed with CUDA events, and
the two routes alternate window by window (R windows each, medians reported, every window listed).  A KITTI frame
keeps its calibration (a sequence), so neither route recomputes the indices; NYU recomputes them every frame in both.
Also reported: the model file's size and the load time (occd_model_load, host clock).  The card's name, power limit
and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


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
    ap.add_argument("names", nargs="*", default=list(sc.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("deploy_bench.py measures on a CUDA (sm_90a) device; none is visible")
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from occdepth_b200 import deploy
    gpu, power = sc.card()
    try:
        clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        clock = "unknown"
    tmp = tempfile.mkdtemp(prefix="occd_deploy_bench_")
    for name in a.names:
        m, _, _ = sc.make_case(name)
        m = m.cuda()
        nyu = sc.CONFIGS[name]["dataset"] == "NYU"
        if nyu:
            frame = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
        else:
            H, W = sc.KITTI_IMG
            frame = dict(kitti_frame(sc.CONFIGS[name]["views"], H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
        frame["img"] = torch.from_numpy(frame["img"]).cuda()      # both routes read device images
        if nyu:
            frame["depth"] = torch.from_numpy(frame["depth"]).cuda()
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            path = os.path.join(tmp, "%s_%s.occd" % (name, prec))
            with torch.no_grad():
                deploy.export(m, path, frame)
                t0 = time.perf_counter()
                cm = deploy.LoadedModel(path)
                torch.cuda.synchronize()
                load_s = time.perf_counter() - t0
                out = torch.empty(1, cm.geom.X, cm.geom.Y, cm.geom.Z, dtype=torch.uint16, device="cuda")
                routes = {"predict_frame": lambda: m.predict_frame(frame),
                          "occd_model_run_frame": lambda: cm.run_frame(frame, out=out)}
                for fn in routes.values():
                    for _ in range(a.warmup):
                        fn()
                ms = {k: [] for k in routes}
                for _ in range(a.windows):
                    for k, fn in routes.items():
                        ms[k].append(_window(fn, a.steps))
                same = torch.equal(m.predict_frame(frame).view(torch.int16), cm.run_frame(frame, out=out).view(torch.int16))
            cm.close()
            size = os.path.getsize(path)
            os.remove(path)
            print(json.dumps(dict(
                config=name, precision=prec,
                predict_frame_ms=round(statistics.median(ms["predict_frame"]), 3),
                run_frame_ms=round(statistics.median(ms["occd_model_run_frame"]), 3),
                predict_frame_windows_ms=[round(t, 3) for t in ms["predict_frame"]],
                run_frame_windows_ms=[round(t, 3) for t in ms["occd_model_run_frame"]],
                maps_equal=bool(same), file_mb=round(size / 2 ** 20, 1), load_s=round(load_s, 3),
                steps=a.steps, warmup=a.warmup, gpu=gpu, power_limit=power, sm_clock_now_max=clock)), flush=True)
        del m
        torch.cuda.empty_cache()
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
