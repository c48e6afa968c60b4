#!/usr/bin/env python
"""What a prediction costs when the classifier writes the class map (OccDepth.predict_classes) instead of the logits
that OccDepth.class_map then reduces (forward + class_map), for every shipped configuration in both arithmetic modes.

  python tools/class_map_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [names...]

One JSON line per (configuration, precision): ms per frame of `class_map(model(batch)["ssc_logit"])`, of
`predict_classes(batch)` and of `predict_classes(batch, confidence=True)` (CUDA events around K calls after W warm-up
calls; R windows, alternating the three, the median is reported and every window listed), the maps compared bit for
bit, and the card's name and power limit read in the same run.  For the configurations whose inputs are the image, the
indices and the FOV masks only (the flosp models), also the serving.FramePipeline figure from pinned host frames to the
host result, with and without classes=True.  For the two released models, also serving.CameraPipeline from uint8
camera frames in host memory to the host class map, without and with confidence=True.  Inputs as in
tools/shipped_configs.py.
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


def _pipeline(m, batch, classes, steps, warmup):
    """ms per frame of FramePipeline over pinned host frames (submit + result of the frame before), end to end"""
    import time
    import torch
    from occdepth_b200.serving import FramePipeline
    img = batch["img"].cpu().pin_memory()
    pix = batch["projected_pix_2"][0].cpu().pin_memory()
    fov = batch["fov_mask_2"][0].cpu().pin_memory()
    pipe = FramePipeline(m, img.shape, pix.shape, fov.shape, classes=classes)
    for _ in range(warmup):
        t = pipe.submit(img, pix, fov)
        if t is not None:
            pipe.result(t)
    pipe.result(pipe.flush())
    t0 = time.perf_counter()
    for _ in range(steps):
        t = pipe.submit(img, pix, fov)
        if t is not None:
            pipe.result(t)
    pipe.result(pipe.flush())
    return (time.perf_counter() - t0) * 1e3 / steps


RELEASED = ("nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti")


def _camera_pipeline(m, name, confidence, steps, warmup):
    """ms per frame of CameraPipeline over three alternating host camera frames (submit + result of the frame before)"""
    import time
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from shipped_configs import CONFIGS, KITTI_FULL, KITTI_IMG, NYU_IMG
    from occdepth_b200.serving import CameraPipeline
    if CONFIGS[name]["dataset"] == "NYU":
        frames, hw = [nyu_frame(1 + i) for i in range(3)], NYU_IMG
    else:
        hw = KITTI_IMG
        frames = [dict(kitti_frame(CONFIGS[name]["views"], hw[0], hw[1], 1 + i), **kitti_geometry(hw[0], hw[1], KITTI_FULL))
                  for i in range(3)]
    pipe = CameraPipeline(m, img_hw=hw, confidence=confidence)
    for i in range(warmup):
        t = pipe.submit(frames[i % 3])
        if t is not None:
            pipe.result(t)
    pipe.result(pipe.flush())
    t0 = time.perf_counter()
    for i in range(steps):
        t = pipe.submit(frames[i % 3])
        if t is not None:
            pipe.result(t)
    pipe.result(pipe.flush())
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    from shipped_configs import CONFIGS, card, make_case, to_cuda
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import gc
    import torch
    if not torch.cuda.is_available():
        sys.exit("class_map_bench.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = card()
    for name in a.names:
        m, batch, _ = make_case(name)
        m = m.cuda()
        b = to_cuda(batch)
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            with torch.no_grad():
                logits_path = lambda: m.class_map(m(b)["ssc_logit"])      # noqa: E731
                fused_path = lambda: m.predict_classes(b)                 # noqa: E731
                conf_path = lambda: m.predict_classes(b, confidence=True)   # noqa: E731
                want = logits_path().view(torch.int16)
                same = bool(torch.equal(want, fused_path().view(torch.int16)))
                same_conf = bool(torch.equal(want, conf_path()[0].view(torch.int16)))
                # the class-map plan cache holds one plan: the fused and confidence columns each get a model copy
                # that shares the weights, so that alternating them times the plans and not their rebuilds
                import copy
                mc = copy.copy(m)
                mc.__dict__["_class_plan_cache"] = {}
                conf_path = lambda: mc.predict_classes(b, confidence=True)   # noqa: E731
                for _ in range(a.warmup):
                    logits_path()
                    fused_path()
                    conf_path()
                ms_l, ms_c, ms_k = [], [], []
                for _ in range(a.repeats):
                    ms_l.append(_window(logits_path, a.steps))
                    ms_c.append(_window(fused_path, a.steps))
                    ms_k.append(_window(conf_path, a.steps))
                line = dict(config=name, precision=prec,
                            ms_forward_class_map=round(statistics.median(ms_l), 3),
                            ms_predict_classes=round(statistics.median(ms_c), 3),
                            ms_predict_classes_conf=round(statistics.median(ms_k), 3),
                            windows_forward_class_map=[round(t, 3) for t in ms_l],
                            windows_predict_classes=[round(t, 3) for t in ms_c],
                            windows_predict_classes_conf=[round(t, 3) for t in ms_k],
                            bit_identical=same and same_conf, steps=a.steps, warmup=a.warmup, repeats=a.repeats)
                if CONFIGS[name]["trans_2d_to_3d"] == "flosp" and CONFIGS[name]["dataset"] == "kitti":
                    e_l, e_c = [], []
                    for _ in range(a.repeats):
                        e_l.append(_pipeline(m, b, False, a.steps, a.warmup))
                        e_c.append(_pipeline(m, b, True, a.steps, a.warmup))
                    line.update(e2e_ms_logits=round(statistics.median(e_l), 3),
                                e2e_ms_classes=round(statistics.median(e_c), 3))
                if name in RELEASED:
                    c_m, c_k = [], []
                    for _ in range(a.repeats):
                        c_m.append(_camera_pipeline(m, name, False, a.steps, a.warmup))
                        c_k.append(_camera_pipeline(mc, name, True, a.steps, a.warmup))
                    line.update(camera_ms_classes=round(statistics.median(c_m), 3),
                                camera_ms_classes_conf=round(statistics.median(c_k), 3))
            line.update(gpu=gpu, power_limit=power)
            print(json.dumps(line), flush=True)
            m.invalidate_plans()
            del mc
            gc.collect()
            torch.cuda.empty_cache()
        del m, b
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
