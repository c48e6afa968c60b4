"""Evaluation losses without a GPU: oracle/losses.py against the reference's values (tests/golden/ssc_losses.pt, made
by oracle/gen_ssc_losses.py from the reference's own OccDepth.step), and occdepth_b200.losses' sums-to-losses
functions on the CPU, fed with the kernels' sums restated in numpy, against the same values and the NaN cases."""
import math
import os

import numpy as np
import pytest
import torch

from occdepth_b200 import losses as L
from oracle import losses as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssc_losses.pt")
TOL = 1e-12


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-300)


def oracle_terms(case, dtype=torch.float64):
    """{log name: value} of the oracle on a fixture case, in OccDepth.step's order, total accumulated as there
    (`loss += term`, so a float32 first term keeps the total float32)"""
    sw, out, batch, st = case["switches"], case["out"], case["batch"], case["step_type"]
    o = {k: v.to(dtype) for k, v in out.items()}
    x, t = o["ssc_logit"], batch["target"]
    terms = []
    if sw["context_prior"] and sw["relation_loss"]:
        terms.append(("loss_relation_ce_super", O.crp(o["P_logits"], batch["CP_mega_matrices"])))
    w = torch.tensor(sw["class_weights"], dtype=torch.float32).to(dtype)
    terms.append(("loss_ssc", O.ce_ssc(x, t, w)))
    if sw["cascade_cls"]:
        tocc = t.clone()
        tocc[(tocc != 0) & (tocc != 255)] = 1
        terms.append(("loss_occ", O.ce_ssc(o["occ_logit"], tocc, torch.tensor(sw["class_weights_occ"]).to(dtype))))
    dp = o["depth_pred"][:, 0:1] if sw["use_stereo_depth_gt"] else o["depth_pred"]
    terms.append(("loss_depth", O.depth(batch["gt_depth"].to(dtype), dp, sw["depth"]["downsample_factor"],
                                        sw["depth"]["d_bound"])))
    terms.append(("loss_sem_scal", O.sem_scal(x, t)))
    terms.append(("loss_geo_scal", O.geo_scal(x, t)))
    if st != "test":
        terms.append(("loss_frustums", O.frustum(x, batch["frustums_masks"], batch["frustums_class_dists"])))
    loss = 0
    for _, v in terms:
        loss += v
    return [(st + "/" + k, v) for k, v in terms] + [(st + "/loss", loss)]


@pytest.mark.parametrize("name", ["kitti", "nyu", "nyu_test"])
def test_oracle_matches_the_reference(golden, name):
    case = golden["cases"][name]
    got = oracle_terms(case)
    assert [k for k, _ in got] == [k for k, _, _ in case["f64"]]
    for (k, v), (_, want, kw) in zip(got, case["f64"]):
        assert rel(v, want) <= TOL, (k, float(v), want)
        assert kw == {"on_epoch": True, "sync_dist": True}


# ---- the kernels' sums, restated in numpy (float64) ----------------------------------------------------------------
def np_ssc_sums(x, t, w, occ=None, occ_w=None, masks=None):
    B, C = x.shape[:2]
    x = x.reshape(B, C, -1).astype(np.float64)
    t = t.reshape(B, -1).astype(np.float64)
    S = x.shape[2]
    F = 0 if masks is None else masks.shape[1]
    m = x.max(1, keepdims=True)
    e = np.exp(x - m)
    se = e.sum(1, keepdims=True)
    p = e / se
    lse = (np.log(se) + m)[:, 0]
    known = t != 255
    is_cls = known & (t >= 0) & (t < C) & (t == np.floor(t))
    cls = np.where(is_cls, t, 0).astype(np.int64)
    xg = np.take_along_axis(x, cls[:, None], 1)[:, 0]
    s = np.zeros(6 + 3 * C + F * C)
    s[0] = (w[cls] * (lse - xg))[is_cls].sum()
    s[1] = w[cls][is_cls].sum()
    s[2], s[3] = known.sum(), (known & ~is_cls).sum()
    if occ is not None:
        o = occ.reshape(B, 2, -1).astype(np.float64)
        go = np.where(is_cls & (cls == 0), 0, 1)
        mo = o.max(1)
        lo = mo + np.log(np.exp(o[:, 0] - mo) + np.exp(o[:, 1] - mo))
        xo = np.where(go == 0, o[:, 0], o[:, 1])
        s[4] = (occ_w[go] * (lo - xo))[known].sum()
        s[5] = occ_w[go][known].sum()
    for c in range(C):
        hit = is_cls & (cls == c)
        s[6 + c] = p[:, c][known].sum()
        s[6 + C + c] = p[:, c][hit].sum()
        s[6 + 2 * C + c] = hit.sum()
    if F:
        s[6 + 3 * C:] = np.einsum("bfs,bcs->fc", masks.reshape(B, F, S).astype(np.float64), p).reshape(-1)
    return torch.from_numpy(s)


def np_crp_sums(P, cp):
    x = P.astype(np.float64)
    y = np.swapaxes(cp, 2, 3).astype(np.float64)          # [B, R, M, N]
    sp_neg = np.logaddexp(0, -x)
    sp_pos = np.logaddexp(0, x)
    ax = (0, 2, 3)
    return torch.from_numpy(np.stack([(y * sp_neg).sum(ax), ((1 - y) * sp_pos).sum(ax), y.sum(ax),
                                      (y == 0).sum(ax)], 1))


def np_depth_sums(gt, prob, f, d_bound):
    n, nc, D, h, w = prob.shape
    H, W = gt.shape[-2:]
    g = gt.reshape(n * nc, H, W).astype(np.float64)
    p = prob.reshape(n * nc, D, h, w).astype(np.float64)
    sh, sw = np.float32(H) / np.float32(h * f), np.float32(W) / np.float32(w * f)
    iy = np.minimum(np.floor(np.arange(h * f, dtype=np.float32) * sh).astype(np.int64), H - 1)
    ix = np.minimum(np.floor(np.arange(w * f, dtype=np.float32) * sw).astype(np.int64), W - 1)
    r = g[:, iy][:, :, ix].reshape(n * nc, h, f, w, f)
    r = np.where(r == 0, 1e5, r).min((2, 4))
    b = (r - (d_bound[0] - d_bound[2])) / d_bound[2]
    k = np.where((b < D + 1) & (b >= 0), b, 0).astype(np.int64)
    fg = k >= 1
    onehot = (np.arange(D)[None, :, None, None] == (k - 1)[:, None]).astype(np.float64)
    bce = -(onehot * np.maximum(np.log(p), -100) + (1 - onehot) * np.maximum(np.log1p(-p), -100)).sum(1)
    return torch.tensor([bce[fg].sum(), fg.sum()], dtype=torch.float64)


def from_sums_terms(case):
    sw, out, batch, st = case["switches"], case["out"], case["batch"], case["step_type"]
    C = sw["n_classes"]
    t = batch["target"].numpy()
    masks = torch.stack(batch["frustums_masks"]).numpy()
    occ = out["occ_logit"].numpy() if sw["cascade_cls"] else None
    ow = np.array(sw["class_weights_occ"], dtype=np.float32).astype(np.float64) if occ is not None else None
    s = np_ssc_sums(out["ssc_logit"].numpy(), t, sw["class_weights"].astype(np.float64), occ, ow, masks)
    terms = L.ssc_losses_from_sums(s, C)
    got = {}
    if sw["context_prior"] and sw["relation_loss"]:
        P = out["P_logits"]
        got["loss_relation_ce_super"] = L.crp_loss_from_sums(
            np_crp_sums(P.numpy(), torch.stack(batch["CP_mega_matrices"]).numpy()), P.shape[0] * P.shape[2] * P.shape[3])
    got["loss_ssc"] = terms["ce"]
    if sw["cascade_cls"]:
        got["loss_occ"] = terms["occ_ce"]
    dp = out["depth_pred"][:, 0:1] if sw["use_stereo_depth_gt"] else out["depth_pred"]
    got["loss_depth"] = L.depth_loss_from_sums(np_depth_sums(batch["gt_depth"].numpy(), dp.numpy(),
                                                             sw["depth"]["downsample_factor"], sw["depth"]["d_bound"]))
    got["loss_sem_scal"] = terms["sem_scal"]
    got["loss_geo_scal"] = terms["geo_scal"]
    if st != "test":
        got["loss_frustums"] = L.frustum_loss_from_sums(s[6 + 3 * C:].view(-1, C), torch.stack(batch["frustums_class_dists"]))
    return got


@pytest.mark.parametrize("name", ["kitti", "nyu", "nyu_test"])
def test_losses_from_sums_match_the_reference(golden, name):
    case = golden["cases"][name]
    got = from_sums_terms(case)
    st = case["step_type"]
    for key, want, _ in case["f64"]:
        k = key[len(st) + 1:]
        if k == "loss":
            continue
        v = got.pop(k)
        assert v.dtype == torch.float64 and v.dim() == 0
        # the reference's relation loss is float32 whatever the logits' dtype (its BCE target is labels.float())
        tol = 1e-6 if k == "loss_relation_ce_super" else TOL
        assert rel(v, want) <= tol, (k, float(v), want)
    assert not got


def test_nan_where_the_reference_fails(golden):
    deg = golden["degenerate"]
    case = golden["cases"]["kitti"]
    sw, out = case["switches"], case["out"]
    x = out["ssc_logit"].numpy()
    w = sw["class_weights"].astype(np.float64)
    C = sw["n_classes"]
    for name, d in (("invalid_label", deg["invalid_label"]), ("all_ignored", deg["all_ignored"])):
        s = np_ssc_sums(x, d["target"].numpy(), w)
        terms = L.ssc_losses_from_sums(s, C)
        for k, key in (("ce", "ce"), ("sem_scal", "sem_scal"), ("geo_scal", "geo_scal")):
            want = d[key]
            if isinstance(want, str) or math.isnan(want):    # the reference raised (or returned NaN)
                assert math.isnan(float(terms[k])), (name, k, want)
            else:
                assert rel(terms[k], want) <= TOL, (name, k, float(terms[k]), want)
    assert deg["invalid_label"]["ce"].startswith("raised:")
    assert deg["no_frustum"]["frustums"] == "raised:ZeroDivisionError"
    empty = torch.zeros(16, C, dtype=torch.float64)
    assert math.isnan(float(L.frustum_loss_from_sums(empty, torch.stack(case["batch"]["frustums_class_dists"]))))
    # a relation without a positive entry: pos_weight is inf, the reference's BCE is NaN
    s = torch.tensor([[0.0, 5.0, 0.0, 10.0], [1.0, 2.0, 3.0, 7.0]], dtype=torch.float64)
    assert math.isnan(float(L.crp_loss_from_sums(s, 10)))
    # no foreground depth pixel: max(1, fg) keeps the loss 0
    assert float(L.depth_loss_from_sums(torch.zeros(2, dtype=torch.float64))) == 0.0


def test_bce_one_range():
    x = torch.tensor([0.0, 1e-50, 0.5, 1.0, 1.0 + 1e-12, -1e-12, math.nan], dtype=torch.float64)
    got = L.bce_one(x)
    assert got[0] == 100.0 and got[1] == 100.0 and got[3] == 0.0
    assert abs(float(got[2]) - math.log(2)) < 1e-15
    assert all(math.isnan(float(v)) for v in got[4:])


def test_switch_values(monkeypatch):
    from occdepth_b200.models.OccDepth import OccDepth
    monkeypatch.delenv("OCCDEPTH_EVAL_LOSSES", raising=False)
    assert OccDepth.eval_losses_enabled() is False
    monkeypatch.setenv("OCCDEPTH_EVAL_LOSSES", "1")
    assert OccDepth.eval_losses_enabled() is True
    monkeypatch.setenv("OCCDEPTH_EVAL_LOSSES", "yes")
    with pytest.raises(ValueError):
        OccDepth.eval_losses_enabled()
