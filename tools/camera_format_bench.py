#!/usr/bin/env python
"""What the camera formats cost: the staging kernel (`occd_stage_camera_u8_cl`) per format, CameraPipeline with RGB
frames against NV12 frames rectified on the device, and the host route it replaces (cv2.cvtColor + cv2.remap).

  python tools/camera_format_bench.py [--launches L] [--windows K] [--frames F] [--host-reps R] [--json OUT]

1. Staging: device time per call for RGB, BGR, NV12 and NV12 + maps, into a tf32 and a bf16 channels-last buffer
   (8 channels), at the KITTI stereo size (2 x 375 x 1242 raw -> 370 x 1220) and NYU's (1 x 480 x 640).  Each
   format's L launches are captured in one CUDA graph, and a window is one replay timed with CUDA events; the formats
   alternate window by window, K windows each, and the median and the range (min, max) are reported.
2. CameraPipeline of the two released models (tf32): ms per frame over F frames after 3 warm-up frames (host clock
   around submits that end in a synchronise), and `h2d_bytes`, for RGB frames and for NV12 frames with rectification
   maps.
3. The host route on this machine's CPU: cv2.cvtColor(NV12 -> RGB) + cv2.remap(INTER_LINEAR) of one KITTI stereo
   frame, ms over R repetitions, with OpenCV's default thread count and with one thread.
One JSON line per measurement, with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

RELEASED = ("nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti")
SIZES = {"kitti_stereo": (2, 375, 1242, 370, 1220), "nyu": (1, 480, 640, 480, 640)}
DIST = (-0.22, 0.06, 0.0008, -0.0011, 0.0)


def rect_maps(V, H, W, f):
    import cv2
    import numpy as np
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]])
    mx, my = cv2.initUndistortRectifyMap(K, np.array(DIST), None, K, (W, H), cv2.CV_32FC1)
    return np.stack([np.stack([mx, my])] * V).astype(np.float32)


def staging(launches, repeats, emit):
    import statistics
    import numpy as np
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200 import data as D
    g = np.random.default_rng(0)
    for size, (V, H0, W0, H, W) in SIZES.items():
        rgb = torch.from_numpy(g.integers(0, 256, size=(V, H0, W0, 3), dtype=np.uint8)).cuda()
        H0e, W0e = H0 + H0 % 2, W0 + W0 % 2
        nv12 = torch.from_numpy(g.integers(0, 256, size=(V, H0e * 3 // 2, W0e), dtype=np.uint8)).cuda()
        maps = torch.from_numpy(rect_maps(V, H, W, 0.58 * W)).cuda()
        for prec, dt, ldt in (("tf32", torch.float32, _lib.DTYPE_F32), ("bf16", torch.bfloat16, _lib.DTYPE_BF16)):
            out = torch.empty(V, H, W, 8, dtype=dt, device="cuda")
            # each format's `launches` calls captured in one CUDA graph: a replay times the kernels back to back on
            # the device, without the host's per-call cost
            graphs = {}
            for fmt, img, mp in (("rgb", rgb, None), ("bgr", rgb, None), ("nv12", nv12, None),
                                 ("nv12+maps", nv12, maps)):
                pf = fmt.split("+")[0]
                fn = (lambda: D.stage_rgb_u8(img, out, ldt, H, W)) if fmt == "rgb" else \
                    (lambda: D.stage_camera_u8(img, out, ldt, H, W, pf, mp))
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    fn()                                      # warm-up outside the capture
                torch.cuda.current_stream().wait_stream(side)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    for _ in range(launches):
                        fn()
                graph.replay()
                graphs[fmt] = graph
            times = {fmt: [] for fmt in graphs}
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(repeats):                          # the formats alternate window by window
                for fmt, graph in graphs.items():
                    torch.cuda.synchronize()
                    e0.record()
                    graph.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times[fmt].append(e0.elapsed_time(e1) * 1000.0 / launches)
            for fmt, t in times.items():
                emit(dict(bench="staging", size=size, precision=prec, format=fmt,
                          us_per_call=round(statistics.median(t), 2), us_min=round(min(t), 2),
                          us_max=round(max(t), 2), launches=launches, windows=repeats, pixels=V * H * W))
            del graphs


def pipeline(frames, emit):
    import numpy as np
    import torch
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from occdepth_b200.serving import CameraPipeline
    for name in RELEASED:
        m, _, _ = sc.make_case(name)
        m = m.cuda().set_precision("tf32")
        nyu = sc.CONFIGS[name]["dataset"] == "NYU"
        if nyu:
            H, W = sc.NYU_IMG
            geo = {}
            fs = [nyu_frame(1 + i) for i in range(frames + 3)]
        else:
            H, W = sc.KITTI_IMG
            geo = {k: v for k, v in kitti_geometry(H, W, sc.KITTI_FULL).items() if k != "img_hw"}
            fs = [kitti_frame(sc.CONFIGS[name]["views"], H, W, 1 + i) for i in range(frames + 3)]
        V, H0, W0 = fs[0]["img"].shape[:3]
        H0e, W0e = H0 + H0 % 2, W0 + W0 % 2
        g = np.random.default_rng(1)
        maps = rect_maps(V, H, W, 0.58 * W)
        for route in ("rgb", "nv12+maps"):
            kw = {} if route == "rgb" else dict(pixel_format="nv12", rect_maps=maps)
            pipe = CameraPipeline(m, img_hw=(H, W), **geo, **kw)
            host = []
            for f in fs:
                f = {k: v for k, v in f.items() if k not in ("vox_origin",) or nyu}
                if route != "rgb":
                    f["img"] = g.integers(0, 256, size=(V, H0e * 3 // 2, W0e), dtype=np.uint8)
                host.append(f)
            with torch.no_grad():
                for f in host[:3]:
                    pipe.submit(f)
                pipe.result(pipe.flush())
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for f in host[3:]:
                    pipe.submit(f)
                pipe.result(pipe.flush())
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1000.0 / frames
            emit(dict(bench="camera_pipeline", model=name, precision="tf32", route=route, ms_per_frame=round(ms, 3),
                      h2d_bytes=pipe.h2d_bytes, frames=frames))
            del pipe
        del m
        torch.cuda.empty_cache()


def host_route(reps, emit):
    import cv2
    import numpy as np
    V, H0, W0, H, W = SIZES["kitti_stereo"]
    g = np.random.default_rng(2)
    nv12 = [g.integers(0, 256, size=((H0 + 1) * 3 // 2, W0), dtype=np.uint8) for _ in range(V)]
    maps = rect_maps(V, H, W, 0.58 * W)
    default = cv2.getNumThreads()
    for threads in (default, 1):
        cv2.setNumThreads(threads)
        for _ in range(3):
            [cv2.remap(cv2.cvtColor(im, cv2.COLOR_YUV2RGB_NV12), mp[0], mp[1], cv2.INTER_LINEAR,
                       borderMode=cv2.BORDER_CONSTANT) for im, mp in zip(nv12, maps)]
        t0 = time.perf_counter()
        for _ in range(reps):
            [cv2.remap(cv2.cvtColor(im, cv2.COLOR_YUV2RGB_NV12), mp[0], mp[1], cv2.INTER_LINEAR,
                       borderMode=cv2.BORDER_CONSTANT) for im, mp in zip(nv12, maps)]
        ms = (time.perf_counter() - t0) * 1000.0 / reps
        emit(dict(bench="host_route", size="kitti_stereo", threads=threads, cpus=os.cpu_count(),
                  ms_per_frame=round(ms, 3), reps=reps))
    cv2.setNumThreads(default)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("camera_format_bench: needs a CUDA device")
    from shipped_configs import card
    gpu, power = card()
    lines = []

    def emit(d):
        d.update(gpu=gpu, power_limit=power)
        lines.append(d)
        print(json.dumps(d), flush=True)
    staging(a.launches, a.windows, emit)
    pipeline(a.frames, emit)
    host_route(a.host_reps, emit)
    if a.json:
        with open(a.json, "w") as fh:
            fh.write("\n".join(json.dumps(d) for d in lines) + "\n")


if __name__ == "__main__":
    main()
