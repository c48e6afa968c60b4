#!/usr/bin/env python
"""Per-rank device time of the X-slab partition of one frame, for every shipped configuration, on ONE card.

  python tools/slab_sim.py [--steps K] [--warmup W] [--repeats N] [--worlds 2,4,8] [--precision tf32|bf16] [names...]

For each configuration (tools/shipped_configs.py, real shapes), precision and world size R, the R rank plans are built
with parallel.SimSlabGroup and each rank's plan is replayed ON ITS OWN (CUDA graph up to the first communication op,
the rest launched eagerly), K replays per window, the median of N windows.  Halo exchanges and all-gathers run as
on-device copies from the peer plans' buffers.  So the figures are per-rank device time of the partitioned plan; they
are not a multi-GPU latency: the NCCL exchange time over NVLink is not in them.  The replay of the unpartitioned plan
is timed the same way.  One JSON line per case:
  ms_per_rank, ms_max (max over ranks), ms_unpartitioned, graph_ops / ops (launches replayed from the graph / all
  launches, per rank), prefix_ms (rank 0's launches before its first communication op, from the per-launch profile:
  the 2-D network -- one view under view sharding -- and, where no all-gather of the views comes first, also the
  virtual view, DepthNet, the lift and the first 1x1x1 conv), depthnet_ms (the replicated DepthNet + softmax of FlospDepth
  configurations, per-launch profile of rank 0), exchanges / exchange_bytes (halo planes sent by the busiest rank per
  forward, both neighbours), gather_bytes (all-gathers received per rank per forward), the card's name and power limit.
A world size the grid does not allow is reported with the partition's refusal.

`rank_plans` / `run_lockstep` are shared with tests/test_gpu_slab_shipped.py.
"""
import argparse
import contextlib
import gc
import io
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _shape_args(m, batch):
    img = batch["img"]
    B, V, _, H, W = img.shape
    pp = batch["projected_pix_%d" % m.project_scale]
    return B, V, H, W, pp[0].shape[1], pp[0].shape[2], img.device


def rank_plans(m, batch, world, capture=False):
    """-> (SimSlabGroup, [plan entry per rank]) for the device batch `batch`; world 1 gives the unpartitioned plan.

    Every rank is built without a CUDA graph: a capture warms up by running the whole plan, and a rank's simulated
    exchanges read peer plans that are not built yet.  With `capture`, each plan is then captured (up to its first
    communication op, as on a real rank) once all its peers exist; a failed capture raises."""
    import torch
    from occdepth_b200.parallel import SimSlabGroup
    B, V, H, W, N, P, dev = _shape_args(m, batch)
    grp = SimSlabGroup(world, halo=3) if world > 1 else None
    ents = []
    saved = os.environ.get("OCCDEPTH_CUDA_GRAPH")
    os.environ["OCCDEPTH_CUDA_GRAPH"] = "0"
    try:
        for r in range(world):
            if grp is not None:
                m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad(), torch.cuda.device(dev), contextlib.redirect_stdout(io.StringIO()):
                ents.append(m._build(B, V, H, W, N, P, dev, batch))
    finally:
        m.__dict__.pop("slab_ctx", None)
        if saved is None:
            os.environ.pop("OCCDEPTH_CUDA_GRAPH")
        else:
            os.environ["OCCDEPTH_CUDA_GRAPH"] = saved
    if capture:
        with torch.no_grad(), torch.cuda.device(dev):
            for e in ents:
                e[0].capture()
                if e[0].graph is None:
                    raise RuntimeError("slab_sim: a rank plan starts with a communication op; nothing to capture")
    return grp, ents


def stage(m, ents, batch):
    ps = m.project_scale
    for e in ents:
        m._stage(e, batch, batch["img"], batch["projected_pix_%d" % ps], batch["fov_mask_%d" % ps],
                 batch["img"].device)


def run_lockstep(m, ents, batch):
    """stage the batch into every rank's plan, run the ranks in lock-step, -> every rank's output dict"""
    import torch
    from occdepth_b200.parallel import SimSlabGroup
    stage(m, ents, batch)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    torch.cuda.synchronize()
    return [m._outputs(e) for e in ents]


def time_plan(plan, steps, warmup, repeats):
    import torch
    for _ in range(warmup):
        plan.run()
    res = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            plan.run()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / steps)
    return statistics.median(res)


def main():
    ap = argparse.ArgumentParser()
    from shipped_configs import CONFIGS, card, make_case, to_cuda
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("slab_sim.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = card()
    for name in a.names:
        m, batch, _ = make_case(name)
        m = m.cuda()
        b = to_cuda(batch)
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            _, (ent,) = rank_plans(m, b, 1, capture=True)
            stage(m, [ent], b)
            ms_full = time_plan(ent[0], a.steps, a.warmup, a.repeats)
            del ent
            gc.collect()            # plans hold reference cycles (ops <-> plan): free their buffers now
            for world in [int(w) for w in a.worlds.split(",")]:
                line = dict(config=name, precision=prec, world=world, ms_unpartitioned=round(ms_full, 3),
                            gpu=gpu, power_limit=power, steps=a.steps, warmup=a.warmup, repeats=a.repeats)
                try:
                    grp, ents = rank_plans(m, b, world, capture=True)
                except NotImplementedError as e:
                    line["refused"] = str(e)
                    print(json.dumps(line), flush=True)
                    continue
                stage(m, ents, b)
                ms = [time_plan(e[0], a.steps, a.warmup, a.repeats) for e in ents]
                prof = ents[0][0].profile()
                ex = [[op for op in e[0].ops if getattr(op, "name", "") == "halo_exchange"] for e in ents]
                ag = [[op for op in e[0].ops if getattr(op, "name", "") == "all_gather"] for e in ents]
                line.update(ms_per_rank=[round(t, 3) for t in ms], ms_max=round(max(ms), 3),
                            graph_ops=[e[0].graph_ops for e in ents], ops=[len(e[0].ops) for e in ents],
                            bounds=grp.ctxs[0].bounds,
                            prefix_ms=round(sum(t for _, t, _ in prof[:ents[0][0].graph_ops]), 3),
                            depthnet_ms=round(sum(t for n, t, _ in prof if n.startswith(("depthnet", "depth."))), 3),
                            exchanges=len(ex[0]),
                            exchange_bytes=max(sum(op.bytes // 2 * ((r > 0) + (r < world - 1)) for op in x)
                                               for r, x in enumerate(ex)),
                            gather_bytes=sum(op.dst.numel() * op.dst.element_size() for op in ag[0]))
                print(json.dumps(line), flush=True)
                del grp, ents
                gc.collect()
                torch.cuda.empty_cache()
        del m, b
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
