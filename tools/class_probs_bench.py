#!/usr/bin/env python
"""What the class probabilities cost next to the other outputs of a prediction, for every shipped configuration in
both arithmetic modes.

  python tools/class_probs_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [--no-files]
                                    [names...]

One JSON line per (configuration, precision) with ms per frame of four routes, timed in R windows of K calls each
(each after W warm-up calls of its route), the routes alternating inside every round; the median is reported and every
window listed:
  map      predict_classes(batch)
  conf     predict_classes(batch, confidence=True)
  probs    predict_classes(batch, probabilities=True)
  logits   model(batch)["ssc_logit"] (the forward plan's fp32 logits)
plus the bytes a pipeline would read back per frame for each (d2h_bytes).  For the two released models, the same four
outputs through model files (deploy.export of a camera frame, LoadedModel.run_frames; the logits route has no file)
are timed the same way.  The card's name and power limit are read in the same run.  Inputs as in
tools/shipped_configs.py.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

RELEASED = ("nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti")


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


def _alternate(routes, steps, warmup, repeats):
    """routes: name -> callable; `repeats` rounds of one window per route, each window after W warm-up calls of its
    route (a model caches one class-map plan, so switching the request rebuilds it: that happens in the warm-up)"""
    windows = {k: [] for k in routes}
    for _ in range(repeats):
        for k, fn in routes.items():
            for _ in range(max(warmup, 1)):
                fn()
            windows[k].append(_window(fn, steps))
    return {k: round(statistics.median(v), 4) for k, v in windows.items()}, \
        {k: [round(x, 4) for x in v] for k, v in windows.items()}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, limit = [x.strip() for x in out[0].split(",")]
        return name, limit
    except Exception:  # noqa: BLE001 -- the figures are still valid, only unlabelled
        return None, None


def _nbytes(t):
    if isinstance(t, (tuple, list)):
        return sum(_nbytes(x) for x in t)
    return t.numel() * t.element_size()


def _file_routes(m, name, tmp):
    """LoadedModel.run_frames of files exported with the map only, with confidence and with probabilities"""
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from occdepth_b200 import deploy
    spec = sc.CONFIGS[name]
    if spec["dataset"] == "NYU":
        frame = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
    else:
        H, W = sc.KITTI_IMG
        frame = dict(kitti_frame(spec["views"], H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
    files = {}
    for k, kw in (("map", {}), ("conf", dict(confidence=True)), ("probs", dict(probabilities=True))):
        path = os.path.join(tmp, "%s.occd" % k)
        deploy.export(m, path, frame, **kw)
        files[k] = deploy.LoadedModel(path)
    return {"map": lambda: files["map"].run_frames([frame]),
            "conf": lambda: files["conf"].run_frames([frame], conf=True),
            "probs": lambda: files["probs"].run_frames([frame], probs=True)}, files


def main():
    import torch
    import shipped_configs as sc
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(sc.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    ap.add_argument("--no-files", action="store_true", help="skip the model-file routes")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("class_probs_bench: needs a CUDA device")
    card, limit = _card()
    for name in a.names:
        for prec in a.precision or ["tf32", "bf16"]:
            m, batch, _ = sc.make_case(name)
            m = m.cuda().set_precision(prec)
            batch = sc.to_cuda(batch)
            with torch.no_grad():
                outs = {"map": m.predict_classes(batch), "conf": m.predict_classes(batch, confidence=True),
                        "probs": m.predict_classes(batch, probabilities=True), "logits": m(batch)["ssc_logit"]}
                assert torch.equal(outs["probs"][0], outs["map"]) and torch.equal(outs["conf"][0], outs["map"])
                routes = {"map": lambda: m.predict_classes(batch),
                          "conf": lambda: m.predict_classes(batch, confidence=True),
                          "probs": lambda: m.predict_classes(batch, probabilities=True),
                          "logits": lambda: m(batch)["ssc_logit"]}
                ms, windows = _alternate(routes, a.steps, a.warmup, a.repeats)
                res = {"config": name, "precision": prec, "card": card, "power_limit": limit,
                       "ms_per_frame": ms, "windows": windows,
                       "d2h_bytes": {k: _nbytes(v) for k, v in outs.items()}}
                if name in RELEASED and not a.no_files:
                    with tempfile.TemporaryDirectory() as tmp:
                        froutes, files = _file_routes(m, name, tmp)
                        res["model_file_ms_per_frame"], res["model_file_windows"] = _alternate(
                            froutes, a.steps, a.warmup, a.repeats)
                        for f in files.values():
                            f.close()
            print(json.dumps(res), flush=True)
            del m, batch, outs
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
