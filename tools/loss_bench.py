#!/usr/bin/env python
"""Evaluation losses on the device: kernel times, achieved bandwidth, the eager route and the validation step.

  python tools/loss_bench.py [--iters N] [--steps K] [--skip-step]

For the released KITTI model's shapes (256 x 256 x 32 voxels, 20 classes, the cascade head, 64 local frustums, CRP
relation logits [1, 4, 512, 4096], stereo depth 104 bins on a 47 x 172 map from a 376 x 1370 gt) and the released
NYU model's (60 x 36 x 60 voxels, 12 classes, 64 frustums, no cascade head or CRP), one frame each:

  - each loss kernel, timed with CUDA events over N launches of the C entry point (buffers preallocated);
  - the bytes each kernel has to move, from the shapes, over its time, against the H100 SXM data sheet's 3.35 TB/s
    of HBM3 (all three kernels are bandwidth-bound: a few fp32 operations per byte);
  - the eager route: oracle/losses.py in float32 on the device (the reference's arithmetic, restated in torch);
  - the validation step of the released models in tf32 with OCCDEPTH_EVAL_LOSSES off and on, CUDA events around K
    steps.

One JSON line per measurement, each with the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

HBM_TBS = 3.35

SHAPES = {
    "kitti": dict(C=20, grid=(256, 256, 32), F=64, occ=True, crp=(4, 512, 4096), depth=((376, 1370), 104, (47, 172),
                                                                                         [2.0, 54.0, 0.5])),
    "nyu": dict(C=12, grid=(60, 36, 60), F=64, occ=False, crp=None, depth=None),
}


def _inputs(shape, seed=0):
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    C, grid, F = shape["C"], shape["grid"], shape["F"]
    x = torch.randn((1, C) + grid, device="cuda", generator=gen) * 2
    t = torch.randint(0, C, (1,) + grid, device="cuda", generator=gen)
    t[torch.rand(t.shape, device="cuda", generator=gen) < 0.6] = 0
    t[torch.rand(t.shape, device="cuda", generator=gen) < 0.1] = 255
    X, Y = grid[:2]
    fid = ((torch.arange(X, device="cuda") * 8 // X)[:, None] * 8
           + (torch.arange(Y, device="cuda") * 8 // Y)[None, :])[:, :, None].expand(grid)
    masks = torch.stack([fid == f for f in range(F)]).unsqueeze(0)
    d = dict(x=x, t=t.float() if shape["occ"] else t.to(torch.uint8), masks=masks,
             dists=torch.randint(0, 300, (1, F, C), device="cuda", generator=gen).float(),
             w=torch.rand(C, device="cuda", generator=gen) + 0.5)
    if shape["occ"]:
        d["occ"] = torch.randn((1, 2) + grid, device="cuda", generator=gen)
        d["w_occ"] = torch.tensor([0.05, 2.0], device="cuda")
    if shape["crp"]:
        R, M, N = shape["crp"]
        d["P"] = torch.randn(1, R, M, N, device="cuda", generator=gen)
        d["cp"] = (torch.rand(1, R, N, M, device="cuda", generator=gen) < 0.2).to(torch.uint8)
    if shape["depth"]:
        (H, W), D, (h, w), db = shape["depth"]
        gt = torch.rand(1, 1, H, W, device="cuda", generator=gen) * 60
        gt[torch.rand(gt.shape, device="cuda", generator=gen) < 0.5] = 0
        d["gt"], d["db"] = gt, db
        d["prob"] = torch.softmax(torch.randn(1, 1, D, h, w, device="cuda", generator=gen), 2)
    return d


def _time(fn, iters, warmup=5):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernels(name, shape, iters, card):
    import torch
    from occdepth_b200 import _lib
    from occdepth_b200 import losses as L
    from oracle import losses as O
    d = _inputs(shape)
    lib, st = _lib.lib(), _lib.stream_ptr()
    C, F = shape["C"], shape["F"]
    S = d["x"][0, 0].numel()
    K = _lib.ssc_loss_sums_len(C, F)
    sums = torch.zeros(K, dtype=torch.float64, device="cuda")
    work = torch.empty(_lib.LOSS_WORK_BLOCKS * K, dtype=torch.float64, device="cuda")
    t = d["t"]
    m8 = d["masks"].view(torch.uint8)
    occ, wocc = d.get("occ"), d.get("w_occ")

    def ssc():
        lib.occd_ssc_loss_sums(d["x"].data_ptr(), t.data_ptr(), L._LABEL_DTYPES[t.dtype], 1, C, S, d["w"].data_ptr(),
                               None if occ is None else occ.data_ptr(), None if wocc is None else wocc.data_ptr(),
                               m8.data_ptr(), F, sums.data_ptr(), work.data_ptr(), work.numel(), st)
    res = []
    ms = _time(ssc, iters)
    nbytes = S * (C * 4 + t.element_size() + F + (8 if occ is not None else 0))
    res.append(dict(kernel="occd_ssc_loss_sums", ms=ms, bytes=nbytes))
    if "P" in d:
        P, cp = d["P"], d["cp"]
        _, R, M, N = P.shape
        cs = torch.zeros(4 * R, dtype=torch.float64, device="cuda")
        cw = torch.empty(_lib.LOSS_WORK_BLOCKS * 4 * R, dtype=torch.float64, device="cuda")
        ms = _time(lambda: lib.occd_crp_relation_sums(P.data_ptr(), cp.data_ptr(), 1, R, M, N, cs.data_ptr(),
                                                      cw.data_ptr(), cw.numel(), st), iters)
        res.append(dict(kernel="occd_crp_relation_sums", ms=ms, bytes=R * M * N * 5))
    if "gt" in d:
        gt, prob, db = d["gt"], d["prob"], d["db"]
        _, _, D, h, w = prob.shape
        H, W = gt.shape[-2:]
        ds = torch.zeros(2, dtype=torch.float64, device="cuda")
        dw = torch.empty(_lib.LOSS_WORK_BLOCKS * 2, dtype=torch.float64, device="cuda")
        ms = _time(lambda: lib.occd_depth_cls_sums(gt.data_ptr(), 1, H, W, prob.data_ptr(), D, h, w, 8, db[0], db[2],
                                                   ds.data_ptr(), dw.data_ptr(), dw.numel(), st), iters)
        fg = int(L.depth_cls_sums(gt, prob, 8, db)[1])
        res.append(dict(kernel="occd_depth_cls_sums", ms=ms, bytes=H * W * 4 + fg * D * 4, fg_pixels=fg))
    for r in res:
        gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9
        print(json.dumps(dict(config=name, **r, us=round(r.pop("ms") * 1e3, 2), gb_per_s=round(gbs, 1),
                              share_of_hbm_datasheet=round(gbs / (HBM_TBS * 1e3), 3), bound="HBM bandwidth",
                              iters=iters, gpu=card[0], power_limit=card[1])), flush=True)

    # the eager route: the reference's arithmetic in float32 on the device, all terms of the validation step
    x = d["x"]
    tt = d["t"]

    def eager():
        O.ce_ssc(x, tt, d["w"])
        if occ is not None:
            to = tt.clone()
            to[(to != 0) & (to != 255)] = 1
            O.ce_ssc(occ, to, wocc)
        O.sem_scal(x, tt)
        O.geo_scal(x, tt)
        O.frustum(x, d["masks"], d["dists"])
        if "P" in d:
            O.crp(d["P"], d["cp"])
        if "gt" in d:
            O.depth(d["gt"], d["prob"], 8, d["db"])

    def fused():
        s = L.ssc_loss_sums(x, tt, d["w"], occ_logits=occ, occ_weight=wocc, frustum_masks=d["masks"])
        L.ssc_losses_from_sums(s, C)
        L.frustum_loss_from_sums(s[6 + 3 * C:].view(-1, C), d["dists"])
        if "P" in d:
            L.crp_loss_from_sums(L.crp_relation_sums(d["P"], d["cp"]), d["P"][0, 0].numel())
        if "gt" in d:
            L.depth_loss_from_sums(L.depth_cls_sums(d["gt"], d["prob"], 8, d["db"]))
    n = max(3, iters // 20)
    ms_e = _time(eager, n, warmup=2)
    ms_f = _time(fused, iters)
    print(json.dumps(dict(config=name, route="all losses of one frame", eager_fp32_ms=round(ms_e, 3),
                          device_sums_ms=round(ms_f, 3), speedup=round(ms_e / ms_f, 1), eager_iters=n, iters=iters,
                          gpu=card[0], power_limit=card[1])), flush=True)


def validation_step(name, steps, card):
    import torch
    import shipped_configs as sc
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_ssc_losses import _eval_batch
    m, batch, _ = sc.make_case(name)
    m = m.cuda()
    batch = sc.to_cuda(batch)
    m.set_precision("tf32")
    if m.cascade_cls:
        m.class_weights_occ = torch.tensor([0.05, 2.0])
    m.log = lambda *a, **k: None
    with torch.no_grad():
        b = _eval_batch(m, batch, m(batch), seed=1)
    res = {}
    for on in ("0", "1", "0", "1"):
        os.environ["OCCDEPTH_EVAL_LOSSES"] = on
        with torch.no_grad():
            ms = _time(lambda: m.validation_step(b, 0), steps, warmup=3)
        res.setdefault(on, []).append(round(ms, 3))
        m.val_metrics.reset()
    os.environ.pop("OCCDEPTH_EVAL_LOSSES", None)
    print(json.dumps(dict(config=name, route="validation_step", precision="tf32", ms_losses_off=res["0"],
                          ms_losses_on=res["1"], steps=steps, gpu=card[0], power_limit=card[1])), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("loss_bench.py measures on a CUDA (sm_90a) device; none is visible")
    import shipped_configs as sc
    card = sc.card()
    for name, shape in SHAPES.items():
        kernels(name, shape, a.iters, card)
        torch.cuda.empty_cache()
    if not a.skip_step:
        for name in ("kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti"):
            validation_step(name, a.steps, card)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
