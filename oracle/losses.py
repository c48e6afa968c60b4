"""Torch restatement of the reference's six loss functions (occdepth/loss/ssc_loss.py, CRP_loss.py, depth_loss.py and
the frustum loss inlined in OccDepth.step).  Device- and dtype-generic: the tests run it in float64 as the comparator
of occdepth_b200.losses, tools/loss_bench.py runs it in float32 on the GPU as the eager route.  Where the reference
can only fail (see occdepth_b200.losses), this restatement fails or returns NaN as torch does; it is compared only
on inputs where the reference returns a value."""
import torch
import torch.nn.functional as F


def _bce_one(x):
    return F.binary_cross_entropy(x, torch.ones_like(x))


def ce_ssc(pred, target, class_weights):
    """CE_ssc_loss: weighted cross-entropy, 255 ignored, mean over the weights of the counted voxels"""
    return F.cross_entropy(pred, target.long(), weight=class_weights.to(pred), ignore_index=255)


def sem_scal(pred, target):
    """sem_scal_loss: per class present among the known voxels, BCE-to-1 of precision, recall and specificity"""
    p = F.softmax(pred, dim=1)
    C = p.shape[1]
    known = target != 255
    pk = p.movedim(1, -1)[known]                                     # [V, C]
    hit = (target[known].unsqueeze(1) == torch.arange(C, device=p.device)).to(p.dtype)
    n_hit, p_sum, p_hit = hit.sum(0), pk.sum(0), (pk * hit).sum(0)
    n_miss, spec_num = (1 - hit).sum(0), ((1 - pk) * (1 - hit)).sum(0)
    loss, count = 0, 0
    for c in range(C):
        if n_hit[c] > 0:
            count += 1
            term = 0
            if p_sum[c] > 0:
                term = term + _bce_one(p_hit[c] / p_sum[c])
            term = term + _bce_one(p_hit[c] / n_hit[c])
            if n_miss[c] > 0:
                term = term + _bce_one(spec_num[c] / n_miss[c])
            loss = loss + term
    return loss / count


def geo_scal(pred, target):
    """geo_scal_loss: BCE-to-1 of the occupied-vs-empty precision, recall and specificity"""
    p = F.softmax(pred, dim=1)[:, 0]
    known = target != 255
    occupied = (target[known] != 0).to(p.dtype)
    empty_p = p[known]
    full_p = 1 - empty_p
    inter = (occupied * full_p).sum()
    return (_bce_one(inter / full_p.sum()) + _bce_one(inter / occupied.sum())
            + _bce_one(((1 - occupied) * empty_p).sum() / (1 - occupied).sum()))


def frustum(pred, frustums_masks, frustums_class_dists):
    """the frustum proportion loss: per local frustum with probability mass and labelled voxels, KL of its class
    proportions (nonzero target classes) against the predicted mass; mean over those frustums.  frustums_masks
    [B, F, ...], frustums_class_dists [B, F, C] (tensors or the batch's lists)"""
    if isinstance(frustums_masks, (list, tuple)):
        frustums_masks = torch.stack(list(frustums_masks))
    if isinstance(frustums_class_dists, (list, tuple)):
        frustums_class_dists = torch.stack(list(frustums_class_dists))
    B, C = pred.shape[:2]
    p = F.softmax(pred, dim=1).reshape(B, C, -1)
    m = frustums_masks.to(p.device).reshape(B, frustums_masks.shape[1], -1).to(p.dtype)
    mass = torch.einsum("bfs,bcs->fc", m, p)
    cnt = frustums_class_dists.to(p.device).float().sum(0)           # float32 counts and proportions, as there
    loss, nonempty = 0, 0
    for f in range(cnt.shape[0]):
        total_cnt, total_prob = cnt[f].sum(), mass[f].sum()
        if total_prob > 0 and total_cnt > 0:
            target = cnt[f] / total_cnt
            keep = target != 0
            loss = loss + F.kl_div(torch.log((mass[f] / total_prob)[keep]), target[keep], reduction="sum")
            nonempty += 1
    return loss / nonempty


def crp(P_logits, CP_mega_matrices):
    """compute_super_CP_multilabel_loss: BCE with logits per relation, pos_weight = #negative / #positive entries.
    P_logits [B, R, M, N] against CP_mega_matrices [B, R, N, M] (tensor or list)"""
    B, R = P_logits.shape[:2]
    logits = P_logits.transpose(2, 3).reshape(B, R, -1).transpose(0, 1).reshape(R, -1).T
    cp = torch.stack(list(CP_mega_matrices)) if isinstance(CP_mega_matrices, (list, tuple)) else CP_mega_matrices
    labels = cp.to(P_logits.device).reshape(B, R, -1).transpose(0, 1).reshape(R, -1).T
    pos_weight = (labels == 0).sum(0) / labels.sum(0)
    return F.binary_cross_entropy_with_logits(logits, labels.float(), pos_weight=pos_weight)


def depth(depth_labels, depth_preds, downsample_factor, d_bound):
    """DepthClsLoss.get_depth_loss: gt [N, n_cam, H, W] against probabilities [N', n_cam', D, h, w]"""
    n, nc, D, h, w = depth_preds.shape
    f = downsample_factor
    H, W = depth_labels.shape[-2:]
    g = depth_labels.reshape(n * nc, 1, H, W).to(depth_preds.device)
    g = F.interpolate(g, (h * f, w * f), mode="nearest").reshape(n * nc, h, f, w, f)
    g = g.permute(0, 1, 3, 2, 4).reshape(n * nc, h, w, f * f)
    g = torch.where(g == 0.0, torch.full_like(g, 1e5), g).min(-1).values
    b = (g - (d_bound[0] - d_bound[2])) / d_bound[2]
    b = torch.where((b < D + 1) & (b >= 0.0), b, torch.zeros_like(b))
    onehot = F.one_hot(b.long(), num_classes=D + 1)[..., 1:].reshape(-1, D).to(depth_preds.dtype)
    p = depth_preds.reshape(n * nc, D, h, w).permute(0, 2, 3, 1).reshape(-1, D)
    fg = onehot.max(1).values > 0
    return F.binary_cross_entropy(p[fg], onehot[fg], reduction="none").sum() / max(1.0, fg.sum())
