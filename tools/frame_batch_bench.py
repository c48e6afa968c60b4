#!/usr/bin/env python
"""Throughput of batched camera frames: ms per frame and frames/s of `OccDepth.predict_frames` and of a batched model
file replayed from C (`occd_model_run_frames`) at B frames per call, per shipped configuration at its shipped shapes.

  python tools/frame_batch_bench.py [--batches 1,2,4,8] [--frames F] [--windows R] [--warmup W] [--no-c]
                                    [--json OUT] [names...]

Every configuration runs in tf32; the two released models (nyu_b4_f100_2080ti, kitti_b3_f32_flospdepth_2080ti) also
in bf16.  For each B both routes run B distinct frames per call on the current stream (KITTI: one calibration per
batch item, as a sequence keeps it; NYU: new poses every frame, so both routes recompute the indices), class map
only.  A window is about F frames (ceil(F / B) calls) after W warm-up calls, timed with CUDA events; the two routes
alternate window by window, R windows each, and the median and the spread (min, max) of ms per frame are reported.
When the C model does not fit beside the Python plan, the Python windows run first, the plan is dropped and the C
windows follow ("alternated": false).
"plan MB" is the device memory the predict_frames plan holds (allocator bytes before and after the build) and
"file MB" what the C model holds (occd_model_info.device_bytes), both also per frame.  The card's name and power
limit are read in the same run.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

RELEASED = ("nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti")


def _window(fn, calls):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _frames(name, n):
    import shipped_configs as sc
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    import numpy as np
    if sc.CONFIGS[name]["dataset"] == "NYU":
        out = []
        for i in range(n):
            f = nyu_frame(1 + i)
            f["cam_pose"] = f["cam_pose"].copy()
            f["cam_pose"][0, 3] += 0.05 * i
            out.append(f)
        return out
    H, W = sc.KITTI_IMG
    geo = kitti_geometry(H, W, sc.KITTI_FULL)
    V = sc.CONFIGS[name]["views"]
    return [dict(kitti_frame(V, H, W, 1 + i, shift=0.1 * (i % 2)), **geo) for i in range(n)]


def bench_case(name, precision, batches, frames_per_window, windows, warmup, with_c):
    import torch
    import shipped_configs as sc
    from occdepth_b200 import deploy
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    frames = _frames(name, max(batches))
    rows = []
    base_ms = None
    for B in batches:
        fr = frames[:B]
        calls = max(1, -(-frames_per_window // B))
        row = dict(config=name, precision=precision, B=B)
        try:
            m.invalidate_plans()
            gc.collect()
            torch.cuda.empty_cache()
            torch.cuda.synchronize()
            td = tempfile.TemporaryDirectory()
            path = os.path.join(td.name, "m.occd")
            with torch.no_grad():
                if with_c:
                    deploy.export(m, path, fr)         # before the Python plan: the export builds a plan of its own
                    gc.collect()
                    torch.cuda.empty_cache()
                a0 = torch.cuda.memory_allocated()
                m.predict_frames(fr)                   # builds (and captures) the B-frame plan
                torch.cuda.synchronize()
                row["plan_MB"] = round((torch.cuda.memory_allocated() - a0) / 2 ** 20, 1)
                run_py = lambda: m.predict_frames(fr)  # noqa: E731
                cm = None
                if with_c:
                    try:
                        cm = deploy.LoadedModel(path)
                    except RuntimeError as e:
                        if "out of memory" not in str(e):
                            raise
                # both routes alternate window by window when both fit on the device; else the Python route's
                # windows run first, its plan is dropped, then the C route's (row "alternated": false)
                row["alternated"] = cm is not None or not with_c
                ms = {"py": []}
                phases = [{"py": run_py}]
                if with_c and cm is not None:
                    phases[0]["c"] = lambda: cm.run_frames(fr, out=out)
                elif with_c:
                    phases.append({"c": lambda: cm.run_frames(fr, out=out)})
                out = torch.empty((B,) + tuple(int(s) for s in m.full_scene_size), dtype=torch.uint16, device="cuda")
                for ph in phases:
                    if "c" in ph and cm is None:
                        m.invalidate_plans()
                        gc.collect()
                        torch.cuda.empty_cache()
                        cm = deploy.LoadedModel(path)
                    for fn in ph.values():
                        for _ in range(warmup):
                            fn()
                    for k in ph:
                        ms.setdefault(k, [])
                    for _ in range(windows):
                        for k, fn in ph.items():
                            ms[k].append(_window(fn, calls) / (calls * B))
                td.cleanup()
                if cm is not None:
                    row["file_MB"] = round(cm.info().device_bytes / 2 ** 20, 1)
                for k, v in ms.items():
                    med = statistics.median(v)
                    row["%s_ms_per_frame" % k] = round(med, 3)
                    row["%s_spread" % k] = [round(min(v), 3), round(max(v), 3)]
                    row["%s_fps" % k] = round(1000.0 / med, 1)
                if cm is not None:
                    cm.close()
            if base_ms is None:
                base_ms = row["py_ms_per_frame"]
            row["py_speedup_vs_B1"] = round(base_ms / row["py_ms_per_frame"], 3)
            row["plan_MB_per_frame"] = round(row["plan_MB"] / B, 1)
            if "file_MB" in row:
                row["file_MB_per_frame"] = round(row["file_MB"] / B, 1)
        except (torch.cuda.OutOfMemoryError, RuntimeError) as e:
            # recorded, not hidden: the next B would not fit either (the library reports its own allocations'
            # failures as RuntimeError)
            if not isinstance(e, torch.cuda.OutOfMemoryError) and "out of memory" not in str(e):
                raise
            row["error"] = "out of memory: %s" % str(e).splitlines()[0]
            rows.append(row)
            print(json.dumps(row), flush=True)
            break
        rows.append(row)
        print(json.dumps(row), flush=True)
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*")
    ap.add_argument("--batches", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=16, help="frames per timed window (rounded up to whole calls)")
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-c", action="store_true", help="skip the model-file route")
    ap.add_argument("--json", default=None, help="also write every row to this file")
    a = ap.parse_args()
    import torch
    import shipped_configs as sc
    if not torch.cuda.is_available():
        raise SystemExit("frame_batch_bench: needs a CUDA (sm_90a) device")
    card, power = sc.card()
    print("card: %s, power limit %s" % (card, power), flush=True)
    names = a.names or list(sc.CONFIGS)
    cases = [(n, "tf32") for n in names] + [(n, "bf16") for n in names if n in RELEASED]
    batches = [int(b) for b in a.batches.split(",")]
    rows = []
    for name, prec in cases:
        rows += bench_case(name, prec, batches, a.frames, a.windows, a.warmup, not a.no_c)
    print("\n%-36s %-5s %2s %10s %16s %8s %10s %10s %9s %9s" % ("config", "prec", "B", "py ms/fr", "py spread",
                                                             "py fr/s", "C ms/fr", "C fr/s", "plan MB", "MB/frame"))
    for r in rows:
        if "error" in r:
            print("%-36s %-5s %2d %s" % (r["config"], r["precision"], r["B"], r["error"]))
            continue
        print("%-36s %-5s %2d %10.3f %16s %8.1f %10s %10s %9.1f %9.1f" % (
            r["config"], r["precision"], r["B"], r["py_ms_per_frame"], "%.3f-%.3f" % tuple(r["py_spread"]),
            r["py_fps"], r.get("c_ms_per_frame", "-"), r.get("c_fps", "-"), r["plan_MB"], r["plan_MB_per_frame"]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=card, power_limit=power, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
