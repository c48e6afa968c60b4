"""Evaluation losses on the device (csrc/losses.cu, occdepth_b200.losses, OccDepth's OCCDEPTH_EVAL_LOSSES hooks):
the fixture cases against the reference's float64 values (tests/golden/ssc_losses.pt), full KITTI / NYU sizes
against oracle/losses.py in float64 on the device for every label dtype, bit-identical sums across runs, NaN for
invalid labels, the C-level refusals, the validation / test hooks of the released models and the slab refusal."""
import math
import os
import types

import pytest
import torch

from occdepth_b200 import _lib
from occdepth_b200 import losses as L
from oracle import losses as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssc_losses.pt")
# fixture cases against the reference's float64 values: twice the largest error measured on an H100 (2.0e-7, the
# depth loss)
TOL_FIXTURE = 4e-7
# full sizes against the float64 oracle
TOL_FULL = 1e-5


def rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-300)


def _model_like(sw):
    """the attributes step_losses reads from an OccDepth, from a fixture case's switches"""
    return types.SimpleNamespace(
        n_classes=sw["n_classes"], context_prior=sw["context_prior"], relation_loss=sw["relation_loss"],
        fp_loss=sw["fp_loss"], CE_ssc_loss=sw["CE_ssc_loss"], sem_scal_loss=sw["sem_scal_loss"],
        geo_scal_loss=sw["geo_scal_loss"], cascade_cls=sw["cascade_cls"], occluded_cls=sw["occluded_cls"],
        class_weights=torch.tensor(sw["class_weights"]),
        class_weights_occ=None if sw["class_weights_occ"] is None else torch.tensor(sw["class_weights_occ"]),
        with_depth_gt=sw["with_depth_gt"], trans_2d_to_3d=sw["trans_2d_to_3d"],
        use_stereo_depth_gt=sw["use_stereo_depth_gt"], depth_downsample_factor=sw["depth"]["downsample_factor"],
        depth_d_bound=sw["depth"]["d_bound"], depth_loss_w=sw["depth_loss_w"], sem_decay_scale=lambda: 1.0)


def _cuda(v):
    if isinstance(v, list):
        return [t.cuda() for t in v]
    return v.cuda() if isinstance(v, torch.Tensor) else v


@pytest.mark.parametrize("name", ["kitti", "nyu", "nyu_test"])
def test_fixture_cases_match_the_reference(name):
    case = torch.load(GOLDEN, weights_only=False)["cases"][name]
    out = {k: v.cuda() for k, v in case["out"].items()}
    batch = {k: _cuda(v) for k, v in case["batch"].items()}
    got = L.step_losses(_model_like(case["switches"]), out, batch, case["step_type"])
    assert list(got) == [k for k, _, _ in case["f64"]]
    errs = {}
    for (k, want, _), v in zip(case["f64"], got.values()):
        assert v.is_cuda and v.dtype == torch.float32 and v.dim() == 0
        errs[k] = rel(v, want)
    print("fixture %s relative errors: %s" % (name, {k: "%.1e" % e for k, e in errs.items()}))
    assert max(errs.values()) <= TOL_FIXTURE, errs


# ---- full sizes -----------------------------------------------------------------------------------------------------
def _full_case(dataset, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    if dataset == "kitti":
        B, C, grid, F, (R, M, N) = 2, 20, (256, 256, 32), 64, (4, 512, 4096)
        (H, W), D, (h, w), d_bound = (376, 1370), 104, (47, 172), [2.0, 54.0, 0.5]
    else:
        B, C, grid, F, (R, M, N) = 2, 12, (60, 36, 60), 64, (4, 1620, 15 * 9 * 15)
        (H, W), D, (h, w), d_bound = (480, 640), 125, (60, 80), [0, 10, 0.08]
    x = torch.randn((B, C) + grid, device=dev, generator=gen) * 2
    x[:, 0] += 2.0                                                # mostly empty, as a scene
    t = torch.randint(1, C, (B,) + grid, device=dev, generator=gen)
    t[torch.rand(t.shape, device=dev, generator=gen) < 0.7] = 0
    t[torch.rand(t.shape, device=dev, generator=gen) < 0.1] = 255
    # 8 x 8 local frustums: blocks of the (X, Y) plane, a few voxels in none
    X, Y = grid[:2]
    fx = (torch.arange(X, device=dev) * 8) // X
    fy = (torch.arange(Y, device=dev) * 8) // Y
    fid = (fx[:, None] * 8 + fy[None, :])[:, :, None].expand(grid)
    masks = torch.stack([(fid == f) for f in range(F)]).unsqueeze(0).repeat(B, 1, 1, 1, 1)
    masks &= torch.rand(masks.shape, device=dev, generator=gen) < 0.9
    masks[:, 7] = False                                          # one empty frustum
    dists = torch.randint(0, 500, (B, F, C), device=dev, generator=gen).float()
    dists[:, 7] = 0
    occ = torch.randn((B, 2) + grid, device=dev, generator=gen)
    P = torch.randn(B, R, M, N, device=dev, generator=gen)
    cp = (torch.rand(B, R, N, M, device=dev, generator=gen) < 0.2).to(torch.uint8)
    gt = torch.rand(B, 1, H, W, device=dev, generator=gen) * (d_bound[1] + 8)
    gt[torch.rand(gt.shape, device=dev, generator=gen) < 0.4] = 0
    prob = torch.softmax(torch.randn(B, 1, D, h, w, device=dev, generator=gen), 2)
    w = torch.rand(C, device=dev, generator=gen) * 3 + 0.1
    return dict(x=x, t=t, masks=masks, dists=dists, occ=occ, P=P, cp=cp, gt=gt, prob=prob, w=w, C=C,
                d_bound=d_bound)


@pytest.mark.parametrize("dataset", ["kitti", "nyu"])
def test_full_size_against_the_oracle(dataset):
    c = _full_case(dataset)
    x, t, C = c["x"], c["t"], c["C"]
    w_occ = torch.tensor([0.05, 2.0], device="cuda")
    x64 = x.double()
    tocc = t.clone()
    tocc[(tocc != 0) & (tocc != 255)] = 1
    want = {"ce": O.ce_ssc(x64, t, c["w"].double()), "occ_ce": O.ce_ssc(c["occ"].double(), tocc, w_occ.double()),
            "sem_scal": O.sem_scal(x64, t), "geo_scal": O.geo_scal(x64, t),
            "frustums": O.frustum(x64, c["masks"], c["dists"])}
    del x64
    for dt in (torch.float32, torch.uint8, torch.int64):
        s = L.ssc_loss_sums(x, t.to(dt), c["w"], occ_logits=c["occ"], occ_weight=w_occ, frustum_masks=c["masks"])
        got = L.ssc_losses_from_sums(s, C)
        got["frustums"] = L.frustum_loss_from_sums(s[6 + 3 * C:].view(-1, C), c["dists"])
        assert int(s[3]) == 0 and int(s[2]) == int((t != 255).sum())
        for k, v in want.items():
            assert rel(got[k], v) <= TOL_FULL, (dataset, dt, k, float(got[k]), float(v))
    P, cp = c["P"], c["cp"]
    crp = L.crp_loss_from_sums(L.crp_relation_sums(P, cp), P.shape[0] * P.shape[2] * P.shape[3])
    assert rel(crp, O.crp(P.double(), cp)) <= TOL_FULL
    f = 8
    dl = L.depth_loss_from_sums(L.depth_cls_sums(c["gt"], c["prob"], f, c["d_bound"]))
    assert rel(dl, O.depth(c["gt"].double(), c["prob"].double(), f, c["d_bound"])) <= TOL_FULL


def test_sums_are_bit_identical_across_runs():
    c = _full_case("kitti", seed=3)
    runs = []
    for _ in range(2):
        runs.append((L.ssc_loss_sums(c["x"], c["t"].float(), c["w"], occ_logits=c["occ"],
                                     occ_weight=torch.tensor([0.05, 2.0]), frustum_masks=c["masks"]),
                     L.crp_relation_sums(c["P"], c["cp"]), L.depth_cls_sums(c["gt"], c["prob"], 8, c["d_bound"])))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    # frames compose by addition: a batch of 2 equals its frames added into one buffer
    s = None
    for b in range(2):
        s = L.ssc_loss_sums(c["x"][b:b + 1], c["t"][b:b + 1].float(), c["w"], frustum_masks=c["masks"][b:b + 1],
                            sums=s)
    whole = L.ssc_loss_sums(c["x"], c["t"].float(), c["w"], frustum_masks=c["masks"])
    assert torch.allclose(s, whole, rtol=1e-12, atol=0)


def test_invalid_labels_give_nan():
    C = 20
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(1, C, 64, 64, 8, device="cuda", generator=gen)
    t = torch.randint(0, C, (1, 64, 64, 8), device="cuda", generator=gen).float()
    w = torch.ones(C)
    clean = L.ssc_losses_from_sums(L.ssc_loss_sums(x, t, w), C)
    assert all(math.isfinite(float(v)) for k, v in clean.items() if k != "occ_ce")
    for bad in (20.0, 1.5, float("nan"), -1.0, 254.0):
        tb = t.clone()
        tb.view(-1)[5] = bad
        s = L.ssc_loss_sums(x, tb, w)
        assert int(s[3]) == 1, bad
        got = L.ssc_losses_from_sums(s, C)
        assert math.isnan(float(got["ce"])), bad
        assert math.isfinite(float(got["sem_scal"])) and math.isfinite(float(got["geo_scal"]))
    ti = t.to(torch.int64)
    ti.view(-1)[3] = -3
    assert math.isnan(float(L.ssc_losses_from_sums(L.ssc_loss_sums(x, ti, w), C)["ce"]))
    # every label ignored: no term has a value
    got = L.ssc_losses_from_sums(L.ssc_loss_sums(x, torch.full_like(t, 255.0), w), C)
    assert all(math.isnan(float(got[k])) for k in ("ce", "sem_scal", "geo_scal"))


def test_c_level_refusals():
    Lb = _lib.lib()
    st = _lib.stream_ptr()
    x = torch.zeros(1, 20, 1000, device="cuda")
    lab = torch.zeros(1000, dtype=torch.uint8, device="cuda")
    w = torch.ones(20, device="cuda")
    masks = torch.zeros(1, 65, 1000, dtype=torch.uint8, device="cuda")
    sums = torch.zeros(6 + 3 * 65 + 65 * 65, dtype=torch.float64, device="cuda")
    work = torch.zeros(_lib.LOSS_WORK_BLOCKS * sums.numel(), dtype=torch.float64, device="cuda")

    def ssc(xp=x.data_ptr(), lp=lab.data_ptr(), ld=_lib.DTYPE_U8, C=20, S=1000, wp=w.data_ptr(), mp=None, F=0,
            sp=sums.data_ptr(), wk=work.data_ptr(), wl=work.numel(), occ=None, ow=None):
        return Lb.occd_ssc_loss_sums(xp, lp, ld, 1, C, S, wp, occ, ow, mp, F, sp, wk, wl, st)
    assert ssc(xp=None) == _lib.ERR_ARG and ssc(lp=None) == _lib.ERR_ARG and ssc(wp=None) == _lib.ERR_ARG
    assert ssc(sp=None) == _lib.ERR_ARG and ssc(wk=None) == _lib.ERR_ARG
    assert ssc(C=65) == _lib.ERR_ARG and ssc(C=0) == _lib.ERR_ARG
    assert ssc(mp=masks.data_ptr(), F=65) == _lib.ERR_ARG
    assert ssc(mp=masks.data_ptr(), F=0) == _lib.ERR_ARG and ssc(F=3) == _lib.ERR_ARG
    assert ssc(ld=_lib.DTYPE_BF16) == _lib.ERR_ARG and ssc(ld=_lib.DTYPE_U16) == _lib.ERR_ARG
    assert ssc(occ=x.data_ptr()) == _lib.ERR_ARG                   # occ logits without their weights
    assert ssc(wl=_lib.LOSS_WORK_BLOCKS * (6 + 3 * 20) - 1) == _lib.ERR_ARG
    assert ssc(S=0) == _lib.ERR_ARG
    P = torch.zeros(1, 17, 32, 32, device="cuda")
    cp = torch.zeros(1, 17, 32, 32, dtype=torch.uint8, device="cuda")

    def crp(Pp=P.data_ptr(), cpp=cp.data_ptr(), R=4, wl=work.numel()):
        return Lb.occd_crp_relation_sums(Pp, cpp, 1, R, 32, 32, sums.data_ptr(), work.data_ptr(), wl, st)
    assert crp(Pp=None) == _lib.ERR_ARG and crp(cpp=None) == _lib.ERR_ARG
    assert crp(R=17) == _lib.ERR_ARG and crp(R=0) == _lib.ERR_ARG
    assert crp(wl=_lib.LOSS_WORK_BLOCKS * 16 - 1) == _lib.ERR_ARG
    gt = torch.zeros(1, 64, 64, device="cuda")
    pr = torch.zeros(1, 1025, 8, 8, device="cuda")

    def dep(gp=gt.data_ptr(), D=104, f=8, step=0.5, wl=work.numel()):
        return Lb.occd_depth_cls_sums(gp, 1, 64, 64, pr.data_ptr(), D, 8, 8, f, 2.0, step, sums.data_ptr(),
                                      work.data_ptr(), wl, st)
    assert dep(gp=None) == _lib.ERR_ARG and dep(D=1025) == _lib.ERR_ARG and dep(D=0) == _lib.ERR_ARG
    assert dep(f=0) == _lib.ERR_ARG and dep(step=0.0) == _lib.ERR_ARG and dep(wl=_lib.LOSS_WORK_BLOCKS * 2 - 1) == 1
    torch.cuda.synchronize()
    assert float(sums.abs().sum()) == 0.0                          # nothing was launched
    assert ssc() == 0 and crp() == 0 and dep() == 0
    torch.cuda.synchronize()
    assert float(sums[2]) == 1000.0                                # every voxel known (label 0)


# ---- model level ----------------------------------------------------------------------------------------------------
def _case(name, **kw):
    from test_gpu_class_map import _case as case
    return case(name, **kw)


def _eval_batch(m, batch, out, seed):
    """the loss inputs a data pipeline adds to a batch: target, CP_mega_matrices, local frustums, a gt depth map"""
    X, Y, Z = (int(s) for s in m.full_scene_size)
    C = m.n_classes
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, C, (1, X, Y, Z), generator=g)
    t[torch.rand(t.shape, generator=g) < 0.7] = 0
    t[torch.rand(t.shape, generator=g) < 0.1] = 255
    b = dict(batch, target=(t.float() if m.dataset == "kitti" else t.to(torch.uint8)).cuda())
    F = m.frustum_size ** 2
    fid = ((torch.arange(X)[:, None] * m.frustum_size // X) * m.frustum_size
           + torch.arange(Y)[None, :] * m.frustum_size // Y)[:, :, None].expand(X, Y, Z)
    b["frustums_masks"] = [torch.stack([fid == f for f in range(F)]).cuda()]
    b["frustums_class_dists"] = [torch.randint(0, 300, (F, C), generator=g).float()]
    if "P_logits" in out:
        _, R, M, N = out["P_logits"].shape
        b["CP_mega_matrices"] = [(torch.rand(R, N, M, generator=g) < 0.2).to(torch.uint8).cuda()]
    if m.with_depth_gt and m.trans_2d_to_3d == "flosp_depth":
        H, W = batch["img"].shape[-2:]
        b["gt_depth"] = (torch.rand(1, 1, H, W, generator=g) * 60).cuda()   # V == 2: the stereo path stays
    return b


def _expected(m, out, b, step_type):
    """(name, value) of oracle/losses.py in float64 on the forward outputs, in OccDepth.step's order"""
    x, t = out["ssc_logit"].double(), b["target"]
    terms = []
    if m.context_prior and m.relation_loss:
        terms.append(("loss_relation_ce_super", O.crp(out["P_logits"].double(), b["CP_mega_matrices"])))
    terms.append(("loss_ssc", O.ce_ssc(x, t, m.class_weights.double().cuda())))
    if m.cascade_cls:
        tocc = t.clone()
        tocc[(tocc != 0) & (tocc != 255)] = 1
        terms.append(("loss_occ", O.ce_ssc(out["occ_logit"].double(), tocc, m.class_weights_occ.double().cuda())))
    if "gt_depth" in b and m.trans_2d_to_3d == "flosp_depth" and m.with_depth_gt:
        terms.append(("loss_depth", O.depth(b["gt_depth"].double(), out["depth_pred"][:, 0:1].double(),
                                            m.depth_downsample_factor, m.depth_d_bound) * m.depth_loss_w))
    terms.append(("loss_sem_scal", O.sem_scal(x, t)))
    terms.append(("loss_geo_scal", O.geo_scal(x, t)))
    if step_type != "test":
        terms.append(("loss_frustums", O.frustum(x, b["frustums_masks"], b["frustums_class_dists"])))
    terms.append(("loss", sum(float(v) for _, v in terms)))
    return [(step_type + "/" + k, float(v)) for k, v in terms]


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name", ["kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti"])
def test_eval_losses_shipped(name, precision, monkeypatch):
    m, batch = _case(name)
    m.set_precision(precision)
    if m.cascade_cls:
        monkeypatch.setattr(m, "class_weights_occ", torch.tensor([0.05, 2.0]))
    with torch.no_grad():
        out = m(batch)
    b = _eval_batch(m, batch, out, seed=4)
    logged = []
    monkeypatch.setattr(m, "log", lambda key, value, **kw: logged.append((key, value, kw)))
    for step_type in ("val", "test"):
        metric = m.val_metrics if step_type == "val" else m.test_metrics
        step = m.validation_step if step_type == "val" else m.test_step
        metric.reset()
        monkeypatch.delenv("OCCDEPTH_EVAL_LOSSES", raising=False)
        with torch.no_grad():
            step(b, 0)                                          # switch off: the metrics only
        counts_off = metric.counts.clone()
        assert logged == []
        metric.reset()
        monkeypatch.setenv("OCCDEPTH_EVAL_LOSSES", "1")
        with torch.no_grad():
            step(b, 0)
        want = _expected(m, out, b, step_type)
        assert [k for k, _, _ in logged] == [k for k, _ in want]
        assert all(kw == {"on_epoch": True, "sync_dist": True} for _, _, kw in logged)
        for (k, v, _), (_, wv) in zip(logged, want):
            assert v.is_cuda and v.dtype == torch.float32 and v.dim() == 0
            assert rel(v, wv) <= TOL_FULL, (name, precision, k, float(v), wv)
        assert torch.equal(metric.counts, counts_off)
        metric.reset()
        logged.clear()


def test_eval_losses_refuse_the_slab_partition(monkeypatch):
    m, batch = _case("nyu_b4_f100_2080ti")
    monkeypatch.setenv("OCCDEPTH_EVAL_LOSSES", "1")
    m.__dict__["slab_ctx"] = object()
    try:
        with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
            m.validation_step(dict(batch), 0)
    finally:
        m.__dict__.pop("slab_ctx", None)
