#!/usr/bin/env python
"""What a prediction costs when the classifier writes the class map (OccDepth.predict_classes) instead of the logits
that OccDepth.class_map then reduces (forward + class_map), for every shipped configuration in both arithmetic modes.

  python tools/class_map_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [names...]

One JSON line per (configuration, precision): ms per frame of `class_map(model(batch)["ssc_logit"])` and of
`predict_classes(batch)` (CUDA events around K calls after W warm-up calls; R windows, alternating the two, the median
is reported and every window listed), both outputs compared bit for bit, and the card's name and power limit read in
the same run.  For the configurations whose inputs are the image, the indices and the FOV masks only (the flosp
models), also the serving.FramePipeline figure from pinned host frames to the host result, with and without
classes=True.  Inputs as in tools/shipped_configs.py.
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
                same = bool(torch.equal(logits_path().view(torch.int16), fused_path().view(torch.int16)))
                for _ in range(a.warmup):
                    logits_path()
                    fused_path()
                ms_l, ms_c = [], []
                for _ in range(a.repeats):
                    ms_l.append(_window(logits_path, a.steps))
                    ms_c.append(_window(fused_path, a.steps))
                line = dict(config=name, precision=prec,
                            ms_forward_class_map=round(statistics.median(ms_l), 3),
                            ms_predict_classes=round(statistics.median(ms_c), 3),
                            windows_forward_class_map=[round(t, 3) for t in ms_l],
                            windows_predict_classes=[round(t, 3) for t in ms_c],
                            bit_identical=same, steps=a.steps, warmup=a.warmup, repeats=a.repeats)
                if CONFIGS[name]["trans_2d_to_3d"] == "flosp" and CONFIGS[name]["dataset"] == "kitti":
                    e_l, e_c = [], []
                    for _ in range(a.repeats):
                        e_l.append(_pipeline(m, b, False, a.steps, a.warmup))
                        e_c.append(_pipeline(m, b, True, a.steps, a.warmup))
                    line.update(e2e_ms_logits=round(statistics.median(e_l), 3),
                                e2e_ms_classes=round(statistics.median(e_c), 3))
            line.update(gpu=gpu, power_limit=power)
            print(json.dumps(line), flush=True)
            m.invalidate_plans()
            gc.collect()
            torch.cuda.empty_cache()
        del m, b
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
