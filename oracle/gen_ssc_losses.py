"""Generates tests/golden/ssc_losses.pt by running the UNMODIFIED reference loss code on seeded small inputs:
  OCCDEPTH_REFERENCE=<checkout of the original project> python -m oracle.gen_ssc_losses

The reference's own `OccDepth.step` (OccDepth.py:378-533) runs on a stand-in `self` whose forward returns the seeded
outputs and whose `log` records each call, so the fixture holds every loss the step logs, in its order, with the
reference's loss functions (loss/ssc_loss.py, CRP_loss.py, depth_loss.py) and its inline frustum loss.  Each case
runs in float64 and in float32 (inputs stored once, as float32 values); in float64 the depth loss's one-hot target
(which the reference makes float32) follows the prediction's dtype.

  kitti      20 classes, a batch of 2, float32 labels with 255, the cascade head, the CRP relation loss, 16 local
             frustums of which one is empty, and stereo depth supervision (gt 43 x 61: not a multiple of the
             downsample factor 8, with zero and out-of-range depths); the validation step
  nyu        12 classes, uint8 labels, frustums, the NYU depth bins (d_bound [0, 10, 0.08]); the validation step
  nyu_test   the nyu inputs in the test step (no frustum loss)

Degenerate inputs call the reference loss functions one by one and record the value or the exception's type:
  invalid_label (a label 20 of 20 classes), all_ignored (every label 255), no_frustum (every frustum mask empty).
"""
import math
import os

import numpy as np
import torch

from . import ref_import

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ssc_losses.pt")

KITTI_DEPTH = dict(downsample_factor=8, d_bound=[2.0, 54.0, 0.5])
NYU_DEPTH = dict(downsample_factor=8, d_bound=[0, 10, 0.08])


def _labels(rng, shape, C):
    t = rng.integers(1, C, size=shape)
    t[rng.random(shape) < 0.5] = 0
    t[rng.random(shape) < 0.1] = 255
    t.reshape(-1)[:C] = np.arange(C)                   # every class present
    return t


def _frustums(rng, B, F, grid, C, empty):
    """masks [B][F][grid] bool (each voxel in at most one frustum, by blocks) and class counts [B][F][C]"""
    n = int(np.prod(grid))
    idx = (np.arange(n) * F) // n
    masks = np.zeros((B, F, n), dtype=bool)
    for b in range(B):
        perm = rng.permutation(F)
        masks[b, perm[idx], np.arange(n)] = True
        masks[b, :, rng.random(n) < 0.1] = False       # some voxels in no frustum
    if empty is not None:
        masks[:, empty] = False
    dists = rng.integers(0, 40, size=(B, F, C)).astype(np.float32)
    dists[rng.random((B, F, C)) < 0.4] = 0
    if empty is not None:
        dists[:, empty] = 0
    return torch.from_numpy(masks.reshape((B, F) + grid)), torch.from_numpy(dists)


def _depth(rng, B, ncam, H, W, d_bound, D, h, w):
    gt = rng.uniform(d_bound[0], d_bound[1] + 6.0, size=(B, ncam, H, W)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.3] = 0                 # no depth
    gt[rng.random(gt.shape) < 0.05] = d_bound[0] - 1.0   # below the first bin
    logits = rng.normal(size=(B, ncam, D, h, w))
    prob = np.exp(logits) / np.exp(logits).sum(2, keepdims=True)
    return torch.from_numpy(gt), torch.from_numpy(prob.astype(np.float32))


def make_case(name):
    """(switches, out, batch): inputs as float32 / label tensors"""
    if name == "kitti":
        rng = np.random.default_rng(10)
        B, C, grid, F, R, M, N = 2, 20, (16, 16, 4), 16, 4, 8, 32
        sw = dict(context_prior=True, relation_loss=True, CE_ssc_loss=True, cascade_cls=True, occluded_cls=False,
                  with_depth_gt=True, trans_2d_to_3d="flosp_depth", use_stereo_depth_gt=True,
                  use_lidar_depth_gt=False, use_depth_gt=False, sem_scal_loss=True, sem_step_decay_loss=False,
                  geo_scal_loss=True, fp_loss=True, n_classes=C, depth=KITTI_DEPTH, depth_loss_w=1.0,
                  class_weights=rng.uniform(0.2, 3.0, C).astype(np.float32), class_weights_occ=[0.05, 2.0])
        target = torch.from_numpy(_labels(rng, (B,) + grid, C).astype(np.float32))
        out = {"ssc_logit": torch.from_numpy(rng.normal(scale=2.0, size=(B, C) + grid).astype(np.float32)),
               "occ_logit": torch.from_numpy(rng.normal(size=(B, 2) + grid).astype(np.float32)),
               "P_logits": torch.from_numpy(rng.normal(size=(B, R, M, N)).astype(np.float32))}
        D = int((54.0 - 2.0) / 0.5)
        gt, prob = _depth(rng, B, 1, 43, 61, KITTI_DEPTH["d_bound"], D, 5, 7)
        out["depth_pred"] = torch.cat([prob, prob.flip(3)], 1)      # two cameras; the step takes the left one
        masks, dists = _frustums(rng, B, F, grid, C, empty=5)
        batch = {"target": target, "gt_depth": gt, "frustums_masks": list(masks), "frustums_class_dists": list(dists),
                 "CP_mega_matrices": [torch.from_numpy((rng.random((R, N, M)) < 0.3).astype(np.uint8))
                                      for _ in range(B)]}
        return sw, out, batch, "val"
    rng = np.random.default_rng(11)
    B, C, grid, F = 2, 12, (8, 6, 8), 16
    sw = dict(context_prior=False, relation_loss=True, CE_ssc_loss=True, cascade_cls=False, occluded_cls=False,
              with_depth_gt=True, trans_2d_to_3d="flosp_depth", use_stereo_depth_gt=False, use_lidar_depth_gt=False,
              use_depth_gt=True, sem_scal_loss=True, sem_step_decay_loss=False, geo_scal_loss=True, fp_loss=True,
              n_classes=C, depth=NYU_DEPTH, depth_loss_w=1.0,
              class_weights=rng.uniform(0.2, 3.0, C).astype(np.float32), class_weights_occ=None)
    target = torch.from_numpy(_labels(rng, (B,) + grid, C).astype(np.uint8))
    out = {"ssc_logit": torch.from_numpy(rng.normal(scale=2.0, size=(B, C) + grid).astype(np.float32))}
    D = int((10 - 0) / 0.08)
    gt, prob = _depth(rng, B, 1, 37, 45, NYU_DEPTH["d_bound"], D, 5, 6)
    out["depth_pred"] = prob
    masks, dists = _frustums(rng, B, F, grid, C, empty=None)
    batch = {"target": target, "gt_depth": gt, "frustums_masks": list(masks), "frustums_class_dists": list(dists)}
    return sw, out, batch, ("test" if name == "nyu_test" else "val")


class _Step:
    """the attributes OccDepth.step reads, a forward that returns fixed outputs, and a recording log"""

    def __init__(self, sw, out, dtype, refs):
        self.__dict__.update({k: v for k, v in sw.items() if k not in ("depth", "class_weights",
                                                                        "class_weights_occ")})
        self.class_weights = torch.tensor(sw["class_weights"], dtype=torch.float32)
        if sw["class_weights_occ"] is not None:
            self.class_weights_occ = torch.tensor(sw["class_weights_occ"], dtype=torch.float32)
        self.depth_loss_fn = _depth_loss_in(refs.DepthClsLoss, dtype)(**sw["depth"])
        self.cur_batch, self.total_batch = 0, 3834 * 30
        self._out = {k: v.to(dtype) for k, v in out.items()}
        self.logged = []

    def __call__(self, batch):
        return dict(self._out)

    def log(self, key, value, **kw):
        self.logged.append((key, float(value), kw))


def _depth_loss_in(cls, dtype):
    """the reference DepthClsLoss, its one-hot target (exact 0 / 1 values, which the reference returns as float32)
    in the prediction's dtype, so that the float64 run computes its binary cross-entropy in float64"""
    class DepthLoss(cls):
        def _get_downsampled_gt_depth(self, gt_depths):
            return super()._get_downsampled_gt_depth(gt_depths).to(dtype)
    return DepthLoss


class _NoMetric:
    def add_batch(self, *a):
        pass


def _refs():
    ns = ref_import.modules()
    with ref_import.quiet():
        import occdepth.loss.ssc_loss as ssc_loss
        from occdepth.loss.depth_loss import DepthClsLoss
    ns.ssc_loss, ns.DepthClsLoss = ssc_loss, DepthClsLoss
    return ns


def _run_step(refs, name, dtype):
    sw, out, batch, step_type = make_case(name)
    me = _Step(sw, out, dtype, refs)
    b = dict(batch, img=torch.zeros(len(batch["target"]), 1, dtype=dtype))
    if "gt_depth" in b:
        b["gt_depth"] = b["gt_depth"].to(dtype)
    refs.OccDepth.OccDepth.step(me, b, step_type, _NoMetric())
    return me.logged


def _outcome(fn):
    try:
        v = float(fn())
        return v
    except (RuntimeError, ZeroDivisionError, IndexError) as e:
        return "raised:" + type(e).__name__


def degenerate(refs):
    L = refs.ssc_loss
    sw, out, batch, _ = make_case("kitti")
    x = out["ssc_logit"].double()
    w = torch.tensor(sw["class_weights"], dtype=torch.float64)
    res = {}
    bad = batch["target"].clone()
    bad.view(-1)[7] = 20.0
    res["invalid_label"] = dict(target=bad, ce=_outcome(lambda: L.CE_ssc_loss(x, bad, w)),
                                sem_scal=_outcome(lambda: L.sem_scal_loss(x, bad)),
                                geo_scal=_outcome(lambda: L.geo_scal_loss(x, bad)))
    ign = torch.full_like(batch["target"], 255.0)
    res["all_ignored"] = dict(target=ign, ce=_outcome(lambda: L.CE_ssc_loss(x, ign, w)),
                              sem_scal=_outcome(lambda: L.sem_scal_loss(x, ign)),
                              geo_scal=_outcome(lambda: L.geo_scal_loss(x, ign)))
    # the frustum loss alone, every mask empty
    only_fp = dict(sw, context_prior=False, CE_ssc_loss=False, with_depth_gt=False, sem_scal_loss=False,
                   geo_scal_loss=False)
    me = _Step(only_fp, out, torch.float64, refs)
    empty = [torch.zeros_like(m) for m in batch["frustums_masks"]]
    b = dict(batch, img=torch.zeros(2, 1, dtype=torch.float64), frustums_masks=empty)
    res["no_frustum"] = dict(frustums=_outcome(lambda: refs.OccDepth.OccDepth.step(me, b, "val", _NoMetric())))
    return res


def generate():
    refs = _refs()
    data = {"cases": {}, "degenerate": None}
    for name in ("kitti", "nyu", "nyu_test"):
        sw, out, batch, step_type = make_case(name)
        rec = dict(switches={k: v for k, v in sw.items()}, out=out, batch=batch, step_type=step_type)
        for dtype, key in ((torch.float64, "f64"), (torch.float32, "f32")):
            logged = _run_step(refs, name, dtype)
            assert all(math.isfinite(v) for _, v, _ in logged), (name, logged)
            rec[key] = logged
        data["cases"][name] = rec
    data["degenerate"] = degenerate(refs)
    return data


def main():
    torch.save(generate(), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
