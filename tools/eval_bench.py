#!/usr/bin/env python
"""Cost of evaluation on the device per shipped configuration (tools/shipped_configs.py), at the shipped shapes.

  python tools/eval_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [--host] [names...]

Prints one JSON line per (configuration, precision), with the card's name and power limit read in the same run:
  predict_ms        predict_classes alone, ms per frame
  predict_count_ms  predict_classes + SSCMetrics.add_batch per frame (what OccDepth.test_step does)
  kernel_us         occd_ssc_confusion alone on that frame's class map and target (CUDA events around 200 launches)
  kernel_gbps       its bytes (class map + target, each read once) over kernel_us, and kernel_hbm_share against the
                    H100 SXM data sheet's 3.35 TB/s
Frame times are medians of R windows of K frames after W warm-up frames (every window listed).  The image, indices,
masks and the target (float32 for KITTI, uint8 for NYU: the datasets' label dtypes) are resident on the device.
--host adds the host route as a LOWER BOUND on the reference's metric cost: the logits' device->host copy, np.argmax
and one np.bincount (the reference's SSCMetrics makes three np.where passes per class instead, which is slower).
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_TBPS = 3.35


def _windows(fn, steps, warmup, repeats):
    import torch
    for _ in range(warmup):
        fn()
    res = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / steps)
    return res


def target_for(m, seed=0):
    """seeded labels in the dataset's dtype: ~70 % empty, ~10 % ignored (255)"""
    import torch
    X, Y, Z = (int(s) for s in m.full_scene_size)
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, m.n_classes, (1, X, Y, Z), generator=g)
    t[torch.rand(t.shape, generator=g) < 0.7] = 0
    t[torch.rand(t.shape, generator=g) < 0.1] = 255
    return (t.float() if m.dataset == "kitti" else t.to(torch.uint8)).cuda()


def kernel_time_us(y, target, n_classes, launches=200):
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200.metrics import _LABEL_DTYPES, _PRED_DTYPES
    L = _lib.lib()
    counts = torch.zeros(n_classes ** 2 + 1, dtype=torch.int64, device=y.device)
    args = (y.data_ptr(), _PRED_DTYPES[y.dtype], target.data_ptr(), _LABEL_DTYPES[target.dtype], y.numel(), n_classes,
            counts.data_ptr())
    st = _lib.stream_ptr()
    for _ in range(10):
        _lib.check(L.occd_ssc_confusion(*args, st), "occd_ssc_confusion")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        L.occd_ssc_confusion(*args, st)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def host_route_ms(m, batch, target, frames=3):
    """logits D2H + np.argmax + np.bincount per frame (wall clock; the forward is excluded)"""
    import numpy as np
    import torch
    t_host = target.cpu().numpy()
    res = []
    with torch.no_grad():
        for _ in range(frames):
            logits = m(batch)["ssc_logit"]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            y = np.argmax(logits.cpu().numpy(), axis=1)
            k = t_host != 255
            np.bincount(t_host[k].astype(np.int64) * m.n_classes + y[k], minlength=m.n_classes ** 2)
            res.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(res)


def main():
    ap = argparse.ArgumentParser()
    import shipped_configs as sc
    ap.add_argument("names", nargs="*", default=list(sc.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    ap.add_argument("--host", action="store_true")
    a = ap.parse_args()
    import torch
    from occdepth_b200.metrics import SSCMetrics
    if not torch.cuda.is_available():
        sys.exit("eval_bench.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = sc.card()
    for name in a.names:
        m, batch, _ = sc.make_case(name)
        m = m.cuda()
        b = sc.to_cuda(batch)
        target = target_for(m)
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            metric = SSCMetrics(m.n_classes)
            with torch.no_grad():
                pred_ms = _windows(lambda: m.predict_classes(b), a.steps, a.warmup, a.repeats)
                both_ms = _windows(lambda: metric.add_batch(m.predict_classes(b), target), a.steps, a.warmup,
                                   a.repeats)
                y = m.predict_classes(b)
            us = kernel_time_us(y, target, m.n_classes)
            nbytes = y.numel() * (y.element_size() + target.element_size())
            gbps = nbytes / (us * 1e-6) / 1e9
            rec = dict(config=name, precision=prec, predict_ms=round(statistics.median(pred_ms), 3),
                       predict_count_ms=round(statistics.median(both_ms), 3),
                       predict_windows_ms=[round(t, 3) for t in pred_ms],
                       predict_count_windows_ms=[round(t, 3) for t in both_ms],
                       voxels=y.numel(), label_dtype=str(target.dtype).replace("torch.", ""), kernel_us=round(us, 2),
                       kernel_bytes=nbytes, kernel_gbps=round(gbps, 1),
                       kernel_hbm_share=round(gbps / (HBM_TBPS * 1e3), 3), steps=a.steps, warmup=a.warmup,
                       gpu=gpu, power_limit=power)
            if a.host:
                rec["host_route_lower_bound_ms"] = round(host_route_ms(m, b, target), 1)
            print(json.dumps(rec), flush=True)
        del m, b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
