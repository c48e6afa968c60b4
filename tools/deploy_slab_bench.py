#!/usr/bin/env python
"""Model files under the X-slab partition against the Python route: ms per frame of `occd_model_run_frame` on every
rank (each rank's file exported by deploy.export(..., slab_output="root"), NCCL through the library's communicator)
and of `OccDepth.predict_frame(slab_output="root")` (torch.distributed), on the same frame.

  torchrun --nproc_per_node W tools/deploy_slab_bench.py [--steps K] [--warmup N] [--windows R] [--precision P] [names...]

Run it once per world size W the machine has (2 .. GPUs).  The two routes alternate window by window (R windows each);
a window is K frames after N warm-up frames on the current stream, timed with CUDA events on every rank, and the
slowest rank's time is reported.  A KITTI frame keeps its calibration, so neither route recomputes the indices; NYU
recomputes them every frame in both.  Rank 0 checks that the two routes' maps are equal and prints one JSON line per
configuration with the card's name and power limit.  The files go to a temporary directory.
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
    import shipped_configs as sc
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(sc.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), default="tf32")
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from camera_frames import kitti_frame, kitti_geometry, nyu_frame
    from occdepth_b200 import deploy, parallel
    world, rank, local = parallel.env_world()
    if world < 2 or torch.cuda.device_count() < 1:
        sys.exit("deploy_slab_bench.py runs under torchrun on 2 or more GPUs (world size %d)" % world)
    torch.cuda.set_device(local)
    parallel.init(backend="nccl", device=torch.device("cuda", local))
    gpu, power = sc.card()
    ids = [deploy.Comm.unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    comm = deploy.Comm(ids[0], rank, world)
    tmp = tempfile.mkdtemp(prefix="occd_slab_bench_")
    for name in a.names:
        spec = sc.CONFIGS[name]
        m, _, _ = sc.make_case(name)                      # seeded: equal on every rank
        m = m.cuda().set_precision(a.precision)
        if spec["dataset"] == "NYU":
            f = dict(nyu_frame(1), img_hw=sc.NYU_IMG)
        else:
            H, W = sc.KITTI_IMG
            f = dict(kitti_frame(spec["views"], H, W, 1), **kitti_geometry(H, W, sc.KITTI_FULL))
        m.enable_slab_parallel(parallel.SlabContext(halo=3))
        path = os.path.join(tmp, "%s.r%d.occd" % (name, rank))
        with torch.no_grad():
            deploy.export(m, path, f, slab_output="root")
        cm = deploy.LoadedModel(path, comm)
        out = torch.empty(1, cm.geom.X, cm.geom.Y, cm.geom.Z, dtype=torch.uint16, device="cuda") if rank == 0 else None
        with torch.no_grad():
            py = m.predict_frame(f, slab_output="root")
        c = cm.run_frame(f, out=out)
        torch.cuda.synchronize()
        equal = bool(torch.equal(py.view(torch.int16), c.view(torch.int16))) if rank == 0 else True

        def py_step():
            with torch.no_grad():
                m.predict_frame(f, slab_output="root")

        def c_step():
            cm.run_frame(f, out=out)
        times = {"predict_frame": [], "occd_model_run_frame": []}
        for _ in range(a.windows):
            for key, fn in (("predict_frame", py_step), ("occd_model_run_frame", c_step)):
                for _ in range(a.warmup):
                    fn()
                dist.barrier()
                times[key].append(parallel.max_over_ranks(_window(fn, a.steps), device=torch.device("cuda")))
        if rank == 0:
            print(json.dumps(dict(config=name, precision=a.precision, world=world, gpu=gpu, power_limit=power,
                                  maps_equal=equal, ms_per_frame={k: statistics.median(v) for k, v in times.items()},
                                  windows=times)), flush=True)
        cm.close()
        del m
        torch.cuda.empty_cache()
        os.remove(path)
    comm.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
