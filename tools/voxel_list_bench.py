#!/usr/bin/env python
"""What the occupied-voxel list costs, for every shipped configuration: the device compaction
(`occd_occupied_voxels`) against the host route it replaces.

  python tools/voxel_list_bench.py [--steps K] [--warmup W] [--repeats R] [--precision tf32|bf16] [names...]

One JSON line per (configuration, precision), with the card's name and power limit read in the same run:
  us_kernel            the three launches of occupied_voxels on the model's class map and a 40 % FOV mask, coordinates
                       included (CUDA events around 20*K calls into one reused list)
  kernel_bytes         what they must move, from the shapes: the map (2 B) and the mask (1 B) per voxel once, 18 B per
                       listed row, 8 B per tile twice; `hbm_floor_us` = that over the data sheet's 3.35 TB/s, and
                       `share_of_hbm_floor` = floor / measured; `*_5pct`: the same with 5 % of the map's voxels kept
                       and the rest emptied (seeded), the density of a scene rather than of random weights
  ms_predict_voxels / ms_predict_classes   OccDepth.predict_voxels and predict_classes, inputs resident on the device
                       (CUDA events around K calls, the two alternating window by window)
  ms_pipeline_voxels / ms_pipeline_classes serving.CameraPipeline(output="voxels") and (classes=True) from pinned uint8
                       frames (host clock around K submits + results), with the bytes each reads back per frame
  ms_list_host         the host route from a finished class map on the device: `.cpu()` of the map, then numpy --
                       `(y > 0) & (y < 255)`, the FOV split, `flatnonzero`, and a gather from a voxel-centre table
                       built once (the scripts rebuild that table every frame; a careful consumer would not) --
                       host clock, per frame
  ms_list_device       the same rows from the same map through occupied_voxels + VoxelList.rows() (the counts and the
                       written rows are read back), host clock ending in the read-back
Each timing is the median of R windows (all listed).  Weights and inputs are seeded; the maps of randomly initialised
models are far denser than a trained model's, and the occupied fraction is printed with the numbers.
"""
import argparse
import gc
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet (a 700 W card)


def main():
    from camera_bench import _Loop, _events, _wall
    from shipped_configs import CONFIGS, KITTI_FULL, KITTI_IMG, NYU_IMG, card, make_case
    import camera_frames as T
    ap = argparse.ArgumentParser()
    ap.add_argument("names", nargs="*", default=list(CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--precision", choices=("tf32", "bf16"), action="append")
    a = ap.parse_args()
    import numpy as np
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200.serving import CameraPipeline
    from occdepth_b200.voxels import occupied_voxels
    if not torch.cuda.is_available():
        sys.exit("voxel_list_bench.py measures on a CUDA (sm_90a) device; none is visible")
    gpu, power = card()
    med = lambda v: round(statistics.median(v), 3)      # noqa: E731
    for name in a.names:
        spec = CONFIGS[name]
        nyu = spec["dataset"] == "NYU"
        m, _, _ = make_case(name)
        m = m.cuda()
        if nyu:
            geo, res = dict(img_hw=NYU_IMG), 0.08
            frames = [T.nyu_frame(s) for s in range(2)]
        else:
            geo, res = T.kitti_geometry(KITTI_IMG[0], KITTI_IMG[1], KITTI_FULL), 0.2
            frames = [T.kitti_frame(spec["views"], KITTI_IMG[0], KITTI_IMG[1], s) for s in range(2)]
            frames[1].update(cam_k=frames[0]["cam_k"], T_velo_2_cam=frames[0]["T_velo_2_cam"])
        pinned = [dict(f, img=torch.from_numpy(f["img"]).pin_memory(),
                       **({"depth": torch.from_numpy(f["depth"]).pin_memory()} if "depth" in f else {}))
                  for f in frames]
        batch = T.host_batch(m, frames[0], geo)
        n_vox = int(np.prod(m.full_scene_size))
        mask_h = np.random.default_rng(0).random(n_vox) < 0.4
        mask_d = torch.from_numpy(mask_h).cuda()
        batch["fov_mask_1"] = [mask_d.view(1, -1, 1)]
        shape = tuple(int(s) for s in m.full_scene_size)
        centres = ((np.stack([i.reshape(-1) for i in np.indices(shape)], 1) * res + res / 2)).astype(np.float32)
        for prec in a.precision or ["tf32", "bf16"]:
            m.set_precision(prec)
            line = dict(config=name, precision=prec, voxels=n_vox)
            with torch.no_grad():
                y = m.predict_classes(batch)
                # 1. the kernels alone
                vl = occupied_voxels(y, mask_d, voxel_size=res)
                n_occ = int(vl.counts().sum())
                kern = lambda: occupied_voxels(y, mask_d, voxel_size=res, out=vl)      # noqa: E731
                us_kernel = []
                for _ in range(a.warmup):
                    kern()
                for _ in range(a.repeats):
                    us_kernel.append(_events(kern, 20 * a.steps) * 1e3)
                kernel_bytes = 3 * n_vox + 18 * n_occ + 2 * 4 * _lib.voxel_work_len(1, n_vox)
                floor_us = kernel_bytes / HBM_BYTES_PER_S * 1e6
                line.update(occupied=n_occ, occupied_fraction=round(n_occ / n_vox, 4), us_kernel=med(us_kernel),
                            windows_us_kernel=[round(t, 3) for t in us_kernel], kernel_bytes=kernel_bytes,
                            hbm_floor_us=round(floor_us, 3),
                            share_of_hbm_floor=round(floor_us / statistics.median(us_kernel), 4))
                # the same on a scene-like map: 5 % of the voxels keep their class, the rest are empty
                y_h = y.cpu().numpy()
                y_h[np.random.default_rng(1).random(y_h.shape) >= 0.05] = 0
                y5 = torch.from_numpy(y_h).cuda()
                n5 = int(occupied_voxels(y5, mask_d, voxel_size=res, out=vl).counts().sum())
                kern5 = lambda: occupied_voxels(y5, mask_d, voxel_size=res, out=vl)    # noqa: E731
                us5 = [_events(kern5, 20 * a.steps) * 1e3 for _ in range(a.repeats)]
                bytes5 = kernel_bytes - 18 * (n_occ - n5)
                line.update(occupied_5pct=n5, us_kernel_5pct=med(us5), windows_us_kernel_5pct=[round(t, 3) for t in us5],
                            kernel_bytes_5pct=bytes5,
                            share_of_hbm_floor_5pct=round(bytes5 / HBM_BYTES_PER_S * 1e6 / statistics.median(us5), 4))

                # 2. the list from a finished class map: host route against device route
                def host_list():
                    flat = y.cpu().numpy().reshape(-1)
                    occ = (flat > 0) & (flat < 255)
                    out = []
                    for sel in (occ & mask_h, occ & ~mask_h):
                        idx = np.flatnonzero(sel)
                        rows = np.empty((len(idx), 4), np.float32)
                        rows[:, :3] = centres[idx]
                        rows[:, 3] = flat[idx]
                        out.append(rows)
                    return out

                def device_list():
                    return occupied_voxels(y, mask_d, voxel_size=res, out=vl).rows()
                hr, dr = host_list(), device_list()
                assert all(np.array_equal(h, d) for h, d in zip(hr, dr)), "the two routes disagree"
                ms_host, ms_dev = [], []
                for _ in range(a.repeats):
                    ms_host.append(_wall(host_list, a.steps))
                    ms_dev.append(_wall(device_list, a.steps))
                line.update(ms_list_host=med(ms_host), ms_list_device=med(ms_dev),
                            windows_list_host=[round(t, 3) for t in ms_host],
                            windows_list_device=[round(t, 3) for t in ms_dev],
                            d2h_bytes_list_host=2 * n_vox, d2h_bytes_list_device=8 + 18 * n_occ)
                # 3. the model's calls
                out_pv = m.predict_voxels(batch)
                pv = lambda: m.predict_voxels(batch, out=out_pv)      # noqa: E731
                pc = lambda: m.predict_classes(batch)                 # noqa: E731
                ms_pv, ms_pc = [], []
                for _ in range(a.warmup):
                    pv()
                    pc()
                for _ in range(a.repeats):
                    ms_pc.append(_events(pc, a.steps))
                    ms_pv.append(_events(pv, a.steps))
                line.update(ms_predict_voxels=med(ms_pv), ms_predict_classes=med(ms_pc),
                            windows_predict_voxels=[round(t, 3) for t in ms_pv],
                            windows_predict_classes=[round(t, 3) for t in ms_pc])
                # 4. the camera pipeline
                pipes = {"voxels": CameraPipeline(m, output="voxels", **geo), "classes": CameraPipeline(m, **geo)}
                loops = {k: _Loop(p, pinned, p.submit) for k, p in pipes.items()}
                ms_pipe = {k: [] for k in pipes}
                for lp in loops.values():
                    for _ in range(a.warmup):
                        lp()
                    lp.drain()
                for _ in range(a.repeats):
                    for k, lp in loops.items():
                        ms_pipe[k].append(_wall(lp, a.steps))
                        lp.drain()
                last = pipes["voxels"].result(pipes["voxels"].flush())
                line.update(ms_pipeline_voxels=med(ms_pipe["voxels"]), ms_pipeline_classes=med(ms_pipe["classes"]),
                            windows_pipeline_voxels=[round(t, 3) for t in ms_pipe["voxels"]],
                            windows_pipeline_classes=[round(t, 3) for t in ms_pipe["classes"]],
                            d2h_bytes_pipeline_voxels=pipes["voxels"].d2h_bytes, d2h_bytes_pipeline_classes=2 * n_vox,
                            pipeline_capacity=pipes["voxels"].capacity, pipeline_truncated=bool(last["truncated"]))
            line.update(steps=a.steps, warmup=a.warmup, repeats=a.repeats, gpu=gpu, power_limit=power)
            print(json.dumps(line), flush=True)
            del pipes, loops, vl, out_pv
            m.invalidate_plans()
            gc.collect()
            torch.cuda.empty_cache()
        del m, batch
        gc.collect()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
