"""Losses of the reference's evaluation step on the device (OccDepth.step, occdepth/models/OccDepth.py:378-533).

Three kernels (csrc/losses.cu) accumulate float64 sums in one pass each: the SSC pass (cross-entropy, the sem-scal
and geo-scal sums, the cascade head's cross-entropy and the local-frustum probability mass), the CRP relation pass
and the depth classification pass.  The `*_from_sums` functions form the reference's losses from those sums with
float64 torch ops wherever the sums live: no `.item()`, no host synchronisation, and the reference's data-dependent
branches become `torch.where`.  They are plain torch, so they run on the CPU too.

Where the reference's loss function can only fail, the loss here is NaN:
  - a label outside [0, C) that is not 255, or a float label that is not an integer: `loss_ssc` (and so `loss`) is
    NaN.  The reference's cross-entropy asserts on the device (IndexError on the CPU).  The other terms treat such a
    voxel as the reference's sem_scal_loss / geo_scal_loss do: a known voxel of no class.
  - a binary cross-entropy whose input is outside [0, 1] or NaN, e.g. recall 0/0 when every label is 255, or a
    specificity with no voxel of the class's complement: the reference raises (RuntimeError on the CPU).
  - no class present (sem-scal's `loss / count` with count 0), or no nonempty frustum: ZeroDivisionError there.
  - a relation with no positive entry: pos_weight is inf, and the reference's BCE is NaN as well.
"""
import math
from collections import OrderedDict

import torch

from . import _lib

_LABEL_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.uint8: _lib.DTYPE_U8, torch.int64: _lib.DTYPE_I64}


def _labels(t, dev):
    """labels as one of the dtypes the kernel reads (float32, uint8, int64); other integer / bool types become int64
    and float64 becomes float32 (label values are small integers, so neither changes one)"""
    t = t.to(dev, non_blocking=True)
    if t.dtype not in _LABEL_DTYPES:
        t = t.to(torch.float32 if t.is_floating_point() else torch.int64)
    return t.contiguous()


def _work(n, dev):
    return torch.empty(_lib.LOSS_WORK_BLOCKS * n, dtype=torch.float64, device=dev)


def _fp32(t, what):
    if not (t.is_cuda and t.dtype == torch.float32):
        raise RuntimeError("occdepth_b200.losses: %s must be a CUDA float32 tensor" % what)
    return t.contiguous()


# ---- kernels ------------------------------------------------------------------------------------------------------
def ssc_loss_sums(logits, target, weight, occ_logits=None, occ_weight=None, frustum_masks=None, sums=None):
    """sums of occd_ssc_loss_sums (float64, OCCD_SSC_LOSS_SUMS(C, F) long) of fp32 logits [B, C, *] against labels
    [B, *] (255 = ignore); weight [C].  occ_logits [B, 2, *] / occ_weight [2]: the cascade head's cross-entropy.
    frustum_masks [B, F, *] (bool or uint8): the frustum probability sums.  Adds to `sums` when it is given."""
    x = _fp32(logits, "logits")
    dev = x.device
    B, C = x.shape[:2]
    S = x[0, 0].numel()
    t = _labels(target, dev)
    if t.numel() != B * S:
        raise ValueError("ssc_loss_sums: target must hold one label per voxel")
    w = weight.to(dev, torch.float32).contiguous()
    ow = None if occ_weight is None else occ_weight.to(dev, torch.float32).contiguous()
    ox = None if occ_logits is None else _fp32(occ_logits, "occ_logits")
    if ox is not None and ox.shape != (B, 2) + tuple(x.shape[2:]):
        raise ValueError("ssc_loss_sums: occ_logits must be [B, 2, *] over the same voxels")
    F = 0
    m = None
    if frustum_masks is not None:
        m = frustum_masks.to(dev, non_blocking=True)
        m = (m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)).contiguous()
        F = m.shape[1]
        if m.numel() != B * F * S:
            raise ValueError("ssc_loss_sums: frustum_masks must be [B, F, *] over the same voxels")
    K = _lib.ssc_loss_sums_len(C, F)
    if sums is None:
        sums = torch.zeros(K, dtype=torch.float64, device=dev)
    work = _work(K, dev)
    _lib.check(_lib.lib().occd_ssc_loss_sums(
        x.data_ptr(), t.data_ptr(), _LABEL_DTYPES[t.dtype], B, C, S, w.data_ptr(),
        None if ox is None else ox.data_ptr(), None if ow is None else ow.data_ptr(),
        None if m is None else m.data_ptr(), F, sums.data_ptr(), work.data_ptr(), work.numel(), _lib.stream_ptr()),
        "occd_ssc_loss_sums")
    return sums


def crp_relation_sums(P_logits, CP_mega_matrices, sums=None):
    """[R, 4] float64 sums of occd_crp_relation_sums: P_logits [B, R, M, N] fp32 against the mega-context matrices
    (a [B, R, N, M] tensor or the batch's list of [R, N, M] ones)"""
    x = _fp32(P_logits, "P_logits")
    dev = x.device
    B, R, M, N = x.shape
    cp = CP_mega_matrices
    if isinstance(cp, (list, tuple)):
        cp = torch.stack([c.to(dev, non_blocking=True) for c in cp])
    cp = cp.to(dev, torch.uint8).contiguous()
    if tuple(cp.shape) != (B, R, N, M):
        raise ValueError("crp_relation_sums: CP_mega_matrices must be [B, R, N, M] for P_logits [B, R, M, N]")
    if sums is None:
        sums = torch.zeros(R, 4, dtype=torch.float64, device=dev)
    work = _work(4 * R, dev)
    _lib.check(_lib.lib().occd_crp_relation_sums(x.data_ptr(), cp.data_ptr(), B, R, M, N, sums.data_ptr(),
                                                 work.data_ptr(), work.numel(), _lib.stream_ptr()),
               "occd_crp_relation_sums")
    return sums


def depth_cls_sums(depth_labels, depth_preds, downsample_factor, d_bound, sums=None):
    """[2] float64 sums of occd_depth_cls_sums: gt depth [N, n_cam, H, W] against the depth probabilities
    [N', n_cam', D, h, w] (N * n_cam == N' * n_cam'), D = int((d_bound[1] - d_bound[0]) / d_bound[2])"""
    p = _fp32(depth_preds, "depth_preds")
    dev = p.device
    n, nc, D, h, w = p.shape
    D_conf = int((d_bound[1] - d_bound[0]) / d_bound[2])
    if D != D_conf:
        raise ValueError("depth_cls_sums: depth_preds has %d bins, d_bound gives %d" % (D, D_conf))
    g = depth_labels.to(dev, torch.float32, non_blocking=True).contiguous()
    H, W = g.shape[-2:]
    if g.numel() != n * nc * H * W:
        raise ValueError("depth_cls_sums: one gt depth map per predicted map")
    if sums is None:
        sums = torch.zeros(2, dtype=torch.float64, device=dev)
    work = _work(2, dev)
    _lib.check(_lib.lib().occd_depth_cls_sums(g.data_ptr(), n * nc, H, W, p.data_ptr(), D, h, w, int(downsample_factor),
                                              float(d_bound[0]), float(d_bound[2]), sums.data_ptr(), work.data_ptr(),
                                              work.numel(), _lib.stream_ptr()),
               "occd_depth_cls_sums")
    return sums


# ---- sums -> losses (plain torch, float64) ------------------------------------------------------------------------
def _nan_like(t):
    return torch.full_like(t, math.nan)


def bce_one(x):
    """F.binary_cross_entropy(x, 1) = -max(log x, -100); NaN where the reference raises (x outside [0, 1] or NaN)"""
    return torch.where((x >= 0) & (x <= 1), -torch.clamp(torch.log(x), min=-100.0), _nan_like(x))


def ssc_losses_from_sums(sums, n_classes):
    """{"ce", "occ_ce", "sem_scal", "geo_scal"} from the first 6 + 3C sums of occd_ssc_loss_sums:
    CE_ssc_loss, the cascade head's CE_ssc_loss, sem_scal_loss and geo_scal_loss (loss/ssc_loss.py:16-99)"""
    s = sums.to(torch.float64)
    C = n_classes
    V, invalid = s[2], s[3]
    ce = torch.where(invalid > 0, _nan_like(s[0]), s[0] / s[1])
    occ_ce = s[4] / s[5]
    P, N, n = s[6:6 + C], s[6 + C:6 + 2 * C], s[6 + 2 * C:6 + 3 * C]
    zero = torch.zeros_like(P)
    present = n > 0
    neg = V - n
    prec = torch.where(P > 0, bce_one(N / P), zero)                       # if torch.sum(p) > 0
    rec = bce_one(N / n)
    spec = torch.where(neg > 0, bce_one((neg - (P - N)) / neg), zero)     # sum (1 - p)(1 - [t = c]) / sum (1 - [t = c])
    count = present.sum()
    total = torch.where(present, prec + rec + spec, zero).sum()
    sem = torch.where(count > 0, total / count, _nan_like(total))
    inter = (V - n[0]) - (P[0] - N[0])                                     # geo-scal: nonempty = not class 0
    geo = bce_one(inter / (V - P[0])) + bce_one(inter / (V - n[0])) + bce_one(N[0] / n[0])
    return {"ce": ce, "occ_ce": occ_ce, "sem_scal": sem, "geo_scal": geo}


def frustum_loss_from_sums(frustum_sums, class_dists):
    """the frustum proportion loss (OccDepth.py:490-517) from the [F, C] probability sums and the batch's
    frustums_class_dists [B, F, C].  The target proportions are float32, as the reference forms them, and so is
    F.kl_div's target * log(target) term"""
    fs = frustum_sums.to(torch.float64)
    cnt = class_dists.to(fs.device, torch.float32).sum(0)                 # batch_cnt
    total_cnt = cnt.sum(1)
    prop32 = cnt / total_cnt.unsqueeze(1)
    prop = prop32.to(torch.float64)
    total_prob = fs.sum(1)
    ok = (total_prob > 0) & (total_cnt > 0)
    cum = fs / total_prob.unsqueeze(1)
    kl_c = torch.xlogy(prop32, prop32).to(torch.float64) - prop * torch.log(cum)
    kl = torch.where(prop != 0, kl_c, torch.zeros_like(prop)).sum(1)                                       # KL_sep
    nonempty = ok.sum()
    total = torch.where(ok, kl, torch.zeros_like(kl)).sum()
    return torch.where(nonempty > 0, total / nonempty, _nan_like(total))


def crp_loss_from_sums(sums, n_entries):
    """BCEWithLogitsLoss(pos_weight=#neg / #pos) of compute_super_CP_multilabel_loss (loss/CRP_loss.py:4-25) from
    the [R, 4] sums; n_entries = B * M * N per relation.  pos_weight is the reference's float32 quotient of the
    counts, and the weight of a positive entry is its float32 1 + (pos_weight - 1)"""
    s = sums.to(torch.float64)
    R = s.shape[0]
    pw = s[:, 3].to(torch.float32) / s[:, 2].to(torch.float32)
    lw = ((pw - 1) + 1).to(torch.float64)
    return (lw * s[:, 0] + s[:, 1]).sum() / (R * n_entries)


def depth_loss_from_sums(sums):
    """DepthClsLoss.get_depth_loss: the BCE sum over foreground pixels / max(1, #foreground)"""
    s = sums.to(torch.float64)
    return s[0] / torch.clamp(s[1], min=1.0)


# ---- one step -----------------------------------------------------------------------------------------------------
def step_losses(model, out, batch, step_type):
    """the losses OccDepth.step logs for `step_type` ("train", "val" or "test"), in its order, as an OrderedDict
    {"<step_type>/loss_...": 0-dim float32 tensor on the device, ..., "<step_type>/loss": their sum}, from the forward
    outputs `out` and `batch`.  Which terms appear follows the reference's switches on `model` (relation_loss,
    CE_ssc_loss, cascade_cls, occluded_cls, the depth supervision, sem_scal_loss, geo_scal_loss, fp_loss) and the
    batch keys it tests; the frustum loss is skipped in the test step, as there."""
    ssc = out["ssc_logit"]
    dev = ssc.device
    target = batch["target"]
    C = model.n_classes
    res = OrderedDict()
    parts = []

    def put(name, value, scale=1.0):
        v = value * scale
        parts.append(v)
        res[step_type + "/" + name] = v.to(torch.float32)

    if model.context_prior and model.relation_loss:
        P = out["P_logits"]
        s = crp_relation_sums(P, batch["CP_mega_matrices"])
        put("loss_relation_ce_super", crp_loss_from_sums(s, P.shape[0] * P.shape[2] * P.shape[3]))
    frustums = model.fp_loss and step_type != "test"
    terms = None
    if model.CE_ssc_loss or model.sem_scal_loss or model.geo_scal_loss or frustums:
        occ = model.CE_ssc_loss and model.cascade_cls
        if occ and model.class_weights_occ is None:
            raise ValueError("step_losses: the cascade head's loss needs the model's class_weights_occ")
        masks = torch.stack([m.to(dev, non_blocking=True) for m in batch["frustums_masks"]]) if frustums else None
        sums = ssc_loss_sums(ssc, target, model.class_weights,
                             occ_logits=out["occ_logit"] if occ else None,
                             occ_weight=model.class_weights_occ if occ else None, frustum_masks=masks)
        terms = ssc_losses_from_sums(sums, C)
    if model.CE_ssc_loss:
        put("loss_ssc", terms["ce"])
        if model.cascade_cls:
            put("loss_occ", terms["occ_ce"])
        if model.occluded_cls and "occluded" in batch:
            s = ssc_loss_sums(out["occluded_logit"], batch["occluded"], torch.ones(2))
            put("loss_occluded", ssc_losses_from_sums(s, 2)["ce"])
    if model.with_depth_gt and model.trans_2d_to_3d == "flosp_depth" and "gt_depth" in batch:
        dp = out["depth_pred"]
        if model.use_stereo_depth_gt:
            dp = dp[:, 0:1]                                                   # only the left camera's depth
        s = depth_cls_sums(batch["gt_depth"], dp, model.depth_downsample_factor, model.depth_d_bound)
        put("loss_depth", depth_loss_from_sums(s), model.depth_loss_w)
    if model.sem_scal_loss:
        put("loss_sem_scal", terms["sem_scal"], model.sem_decay_scale())
    if model.geo_scal_loss:
        put("loss_geo_scal", terms["geo_scal"])
    if frustums:
        K0 = 6 + 3 * C
        fs = sums[K0:].view(-1, C)
        dists = torch.stack([d.to(dev, non_blocking=True) for d in batch["frustums_class_dists"]])
        put("loss_frustums", frustum_loss_from_sums(fs, dists))
    total = torch.zeros((), dtype=torch.float64, device=dev)
    for v in parts:
        total = total + v
    res[step_type + "/loss"] = total.to(torch.float32)
    return res
