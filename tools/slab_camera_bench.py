#!/usr/bin/env python
"""Latency of one camera frame under the X-slab partition over NCCL, against the one-GPU camera route.

  torchrun --nproc_per_node R tools/slab_camera_bench.py [--frames K] [--warmup W] [--repeats N]
                                                         [--precision tf32|bf16] [--all] [names...]

Every rank runs `serving.CameraPipeline(model, slab_output="root")` on the same uint8 camera frames (held in host
memory, as a serving loop holds decoded images); rank 0 reads back the whole class map.  A window is K frames submitted
back to back, timed with the host clock between a barrier plus synchronisation before and a synchronisation after; the
slowest rank's window counts.  `ms_per_frame` is the median of N windows, `spread_ms` their max - min.  The same
frames then run through the one-GPU route (`CameraPipeline(model)` without the partition) on rank 0, in the same
session and timed the same way, while the other ranks wait.  Default: the two released models (tf32 and bf16); --all:
every shipped configuration (tools/shipped_configs.py).  One JSON line per case, with `h2d_bytes` per rank (the
bytes one frame copies host -> device on that rank), the slab bounds, the card's name and power limit.  A world size
the grid does not allow is reported with the partition's refusal.  Needs at least two GPUs; there is no fall-back.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

RELEASED = ["kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti"]


def _frames(sc, spec):
    """two frames that alternate: KITTI keeps one calibration (a sequence), NYU moves the camera every frame"""
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    if spec["dataset"] == "NYU":
        frames = [nyu_frame(1), nyu_frame(2)]
        frames[1]["cam_pose"][0, 3] += 0.2
        return frames, dict(img_hw=sc.NYU_IMG)
    H, W = sc.KITTI_IMG
    return ([kitti_frame(spec["views"], H, W, s) for s in (1, 2)], kitti_geometry(H, W, sc.KITTI_FULL))


def _window(pipe, frames, k, dist):
    """seconds for k frames through `pipe`, from a common start to the slowest rank's end"""
    import torch
    from occdepth_b200 import parallel
    if dist:
        parallel.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(k):
        t = pipe.submit(frames[i % len(frames)])
        if t is not None:
            pipe.result(t)
    pipe.result(pipe.flush())
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return parallel.max_over_ranks(dt, torch.device("cuda")) if dist else dt


def _time(pipe, frames, a, dist):
    per_frame = []
    _window(pipe, frames, a.warmup, dist)
    for _ in range(a.repeats):
        per_frame.append(_window(pipe, frames, a.frames, dist) * 1e3 / a.frames)
    return statistics.median(per_frame), max(per_frame) - min(per_frame), per_frame


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*")
    ap.add_argument("--all", action="store_true", help="every shipped configuration, not only the released models")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import torch
    from occdepth_b200 import parallel
    from occdepth_b200.serving import CameraPipeline
    import shipped_configs as sc
    world, rank, local = parallel.env_world()
    if world < 2 or torch.cuda.device_count() < 2:
        sys.exit("slab_camera_bench.py measures the partition over NCCL: run it under torchrun --nproc_per_node R with "
                 "R >= 2 on a machine with at least two GPUs (world size %d, %d GPU(s) visible)"
                 % (world, torch.cuda.device_count()))
    torch.cuda.set_device(local)
    parallel.init(backend="nccl", device=torch.device("cuda", local))
    import torch.distributed as dist
    gpu, power = sc.card()
    names = a.names or (list(sc.CONFIGS) if a.all else RELEASED)
    for name in names:
        spec = sc.CONFIGS[name]
        with contextlib.redirect_stdout(io.StringIO()):
            m, _, _ = sc.make_case(name)
        m = m.cuda()
        frames, geo = _frames(sc, spec)
        for prec in a.precision or ["tf32", "bf16"]:
            m.__dict__.pop("slab_ctx", None)
            m.set_precision(prec)
            line = dict(config=name, precision=prec, world=world, frames=a.frames, warmup=a.warmup,
                        repeats=a.repeats, gpu=gpu, power_limit=power)
            with torch.no_grad():
                if rank == 0:
                    pipe = CameraPipeline(m, **geo)
                    ms1, spread1, _ = _time(pipe, frames, a, False)
                    line.update(one_gpu_ms_per_frame=round(ms1, 3), one_gpu_spread_ms=round(spread1, 3),
                                one_gpu_h2d_bytes=pipe.h2d_bytes)
                    del pipe
                parallel.barrier()
                m.enable_slab_parallel(parallel.SlabContext(halo=3))
                try:
                    pipe = CameraPipeline(m, slab_output="root", **geo)
                    ms, spread, windows = _time(pipe, frames, a, True)
                except parallel.SlabPartitionError as e:
                    line["refused"] = str(e)
                    pipe = None
            if pipe is not None:
                h2d = [None] * world
                dist.all_gather_object(h2d, pipe.h2d_bytes)
                line.update(ms_per_frame=round(ms, 3), spread_ms=round(spread, 3),
                            windows_ms=[round(t, 3) for t in windows], h2d_bytes=h2d,
                            bounds=[(lo * m.project_scale, hi * m.project_scale)
                                    for lo, hi in m.__dict__["slab_ctx"].bounds])
            if rank == 0:
                print(json.dumps(line), flush=True)
            del pipe
            m.invalidate_plans()
            torch.cuda.empty_cache()
        del m
        torch.cuda.empty_cache()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
