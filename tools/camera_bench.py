#!/usr/bin/env python
"""What serving a camera frame costs: uint8 images and calibration in host memory -> class map in host memory, for
every shipped configuration in both arithmetic modes.

  python tools/camera_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [names...]

One JSON line per (configuration, precision), with the card's name, power limit and SM clocks read in the same run:
  ms_camera_pipeline  serving.CameraPipeline(classes=True) from pinned uint8 frames: host clock around K submits +
                      results after W warm-up submits (the images, the NYU depth PNG and the matrices cross PCIe; the
                      normalisation and the indices are computed on the device).  KITTI frames share one calibration
                      (a sequence), so the indices are computed once; NYU poses change every frame.
  ms_predict_classes  OccDepth.predict_classes with every input resident on the device (CUDA events around K calls)
  ms_host_route       the route CameraPipeline replaces, where it exists (the configurations whose inputs are the image,
                      the indices and the FOV masks only): numpy normalisation + the numpy vox2pix
                      (oracle.projection) per view + serving.FramePipeline(classes=True), host clock per frame
  h2d_bytes_*         bytes copied host -> device per frame by each route
Each timing is the median of R windows (all listed).  Inputs are seeded; the time does not depend on the values.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def clocks():
    """current and maximum SM clock (MHz) of the current device, asked by UUID"""
    import torch
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader",
                              "-i", "GPU-%s" % props.uuid], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        out = ""
    return out or "unknown"


def _wall(fn, steps):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def _events(fn, steps):
    import torch
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


class _Loop:
    """submit frames[i % n] and read back the previous frame's result; drain() reads the last one"""

    def __init__(self, pipe, frames, submit):
        self.pipe, self.frames, self.submit, self.i = pipe, frames, submit, 0

    def __call__(self):
        t = self.submit(self.frames[self.i % len(self.frames)])
        self.i += 1
        if t is not None:
            self.pipe.result(t)

    def drain(self):
        self.pipe.result(self.pipe.flush())


def main():
    from shipped_configs import CONFIGS, KITTI_FULL, KITTI_IMG, NYU_IMG, card, make_case
    import camera_frames as T
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import gc
    import torch
    from oracle.projection import vox2pix
    from occdepth_b200.serving import CameraPipeline, FramePipeline
    if not torch.cuda.is_available():
        sys.exit("camera_bench.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = card()
    for name in a.names:
        spec = CONFIGS[name]
        nyu = spec["dataset"] == "NYU"
        m, _, _ = make_case(name)
        m = m.cuda()
        if nyu:
            geo = dict(img_hw=NYU_IMG)
            frames = [T.nyu_frame(s) for s in range(2)]
        else:
            geo = T.kitti_geometry(KITTI_IMG[0], KITTI_IMG[1], KITTI_FULL)
            frames = [T.kitti_frame(spec["views"], KITTI_IMG[0], KITTI_IMG[1], s) for s in range(2)]
            frames[1].update(cam_k=frames[0]["cam_k"], T_velo_2_cam=frames[0]["T_velo_2_cam"])
        pinned = [dict(f, img=torch.from_numpy(f["img"]).pin_memory(),
                       **({"depth": torch.from_numpy(f["depth"]).pin_memory()} if "depth" in f else {}))
                  for f in frames]
        batch = T.host_batch(m, frames[0], geo)
        host_route = spec["trans_2d_to_3d"] == "flosp" and not nyu
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            line = dict(config=name, precision=prec)
            with torch.no_grad():
                pipe = CameraPipeline(m, classes=True, **geo)
                cam = _Loop(pipe, pinned, pipe.submit)
                pred = lambda: m.predict_classes(batch)      # noqa: E731
                for _ in range(a.warmup):
                    cam()
                    pred()
                cam.drain()
                h2d_cam = pipe.h2d_bytes
                ms_cam, ms_pred, ms_host = [], [], []
                if host_route:
                    H, W = geo["img_hw"]
                    ps = m.project_scale
                    b0 = {k: (v.cpu().pin_memory() if torch.is_tensor(v) else [t.cpu().pin_memory() for t in v])
                          for k, v in batch.items() if k in ("img", "projected_pix_%d" % ps, "fov_mask_%d" % ps)}
                    fpipe = FramePipeline(m, b0["img"].shape, b0["projected_pix_%d" % ps][0].shape,
                                          b0["fov_mask_%d" % ps][0].shape, classes=True)
                    stage = [{k: (v.clone().pin_memory() if torch.is_tensor(v) else [t.clone().pin_memory() for t in v])
                              for k, v in b0.items()} for _ in range(2)]

                    def host_submit(f, n=[0]):
                        """the dataset's per-frame work, then the pipeline (a pinned staging set per frame in flight)"""
                        s = stage[n[0] & 1]
                        n[0] += 1
                        imgs = [T.host_img(im, H, W) for im in f["img"].numpy()]
                        s["img"][0].copy_(torch.stack(imgs))
                        for v in range(len(imgs)):
                            p, fv, _ = vox2pix(f["T_velo_2_cam"][v], f["cam_k"][v], geo["vox_origin"],
                                               geo["voxel_size"], W, H, geo["scene_size"], 0)
                            s["projected_pix_%d" % ps][0][v].copy_(torch.from_numpy(p))
                            s["fov_mask_%d" % ps][0][v].copy_(torch.from_numpy(fv))
                        return fpipe.submit(s["img"], s["projected_pix_%d" % ps][0], s["fov_mask_%d" % ps][0])
                    host = _Loop(fpipe, pinned, host_submit)
                    for _ in range(a.warmup):
                        host()
                    host.drain()
                    h2d_host = sum(t.numel() * t.element_size() for t in (b0["img"], b0["projected_pix_%d" % ps][0],
                                                                         b0["fov_mask_%d" % ps][0]))
                for _ in range(a.repeats):
                    ms_cam.append(_wall(cam, a.steps))
                    cam.drain()
                    ms_pred.append(_events(pred, a.steps))
                    if host_route:
                        ms_host.append(_wall(host, a.steps))
                        host.drain()
            line.update(ms_camera_pipeline=round(statistics.median(ms_cam), 3),
                        ms_predict_classes=round(statistics.median(ms_pred), 3),
                        windows_camera_pipeline=[round(t, 3) for t in ms_cam],
                        windows_predict_classes=[round(t, 3) for t in ms_pred], h2d_bytes_camera=h2d_cam)
            if host_route:
                line.update(ms_host_route=round(statistics.median(ms_host), 3),
                            windows_host_route=[round(t, 3) for t in ms_host], h2d_bytes_host_route=h2d_host)
            line.update(steps=a.steps, warmup=a.warmup, repeats=a.repeats, gpu=gpu, power_limit=power,
                        sm_clock_mhz_now_max=clocks())
            print(json.dumps(line), flush=True)
            del pipe
            m.invalidate_plans()
            gc.collect()
            torch.cuda.empty_cache()
        del m, batch
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
