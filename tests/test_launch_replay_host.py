"""tests/launch_replay.py without a GPU: the census of the non-convolution launches the shipped configurations plan
(recorded on CPU), its float64 references against torch's float64 operations, and the sharpness of its comparator on
results corrupted on the host."""
import contextlib
import io
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import launch_replay as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f64 = torch.float64


@pytest.fixture(autouse=True)
def simt(monkeypatch):
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")


def _tools():
    p = os.path.join(ROOT, "tools")
    if p not in sys.path:
        sys.path.insert(0, p)
    import shipped_configs
    import slab_sim
    return shipped_configs, slab_sim


def _record(m, batch, classes=None, slab=None, depth_items=False):
    """(records, storages) of one plan built on CPU"""
    _, slab_sim = _tools()
    B, V, H, W, N, P, dev = slab_sim._shape_args(m, batch)
    if slab is not None:
        m.__dict__["slab_ctx"] = slab
    try:
        with LR.Recording() as R, torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
            plan = m._build(B, V, H, W, N, P, dev, batch, classes=classes, capture=False, depth_items=depth_items)[0]
            recs = R.calls(plan)
    finally:
        m.__dict__.pop("slab_ctx", None)
    return recs, LR.Storages(LR.plan_tensors(plan))


def test_census_of_the_shipped_configurations(capsys):
    """entry points and distinct launches of the six configurations' forward and class-map plans, then of the slab,
    infer-mode and batched-NYU variants; every recorded entry point has a reference and a region spec"""
    from occdepth_b200.parallel import SimSlabGroup
    sc, _ = _tools()
    lines, total, names = [], 0, set()
    variants = []
    for name in sc.CONFIGS:
        m, batch, _ = sc.make_case(name)
        sigs, n = set(), 0
        for classes in (None, ("classes", None)):
            recs, st = _record(m, batch, classes)
            n += len(recs)
            sigs |= {LR.signature(r, st) for r in recs}
            names |= {r[0] for r in recs}
        per = {}
        for s in sigs:
            per[s[0]] = per.get(s[0], 0) + 1
        lines.append("%-40s %4d launches, %4d distinct: %s" % (name, n, len(sigs),
                                                               ", ".join("%s %d" % kv for kv in sorted(per.items()))))
        total += len(sigs)
        if name == "kitti_b3_f32_flospdepth_2080ti":
            recs, st = _record(m, batch, slab=SimSlabGroup(4, halo=3).ctxs[1])
            variants.append(("%s slab rank 1 of 4" % name, recs, st))
        if name == "nyu_b4_f100_2080ti":
            b2 = dict(batch)
            b2["img"] = batch["img"].repeat(2, 1, 1, 1, 1)
            b2["gt_depth"] = batch["gt_depth"].repeat(2, 1, 1, 1)
            b2["projected_pix_1"] = batch["projected_pix_1"] * 2
            b2["fov_mask_1"] = batch["fov_mask_1"] * 2
            recs, st = _record(m, b2, ("classes", None), depth_items=True)
            variants.append(("%s two frames (depth_items)" % name, recs, st))
        del m, batch
    m, batch, _ = sc.make_case("kitti_b3_f24_flospdepth_mono_2080ti", infer_mode=True)
    recs, st = _record(m, batch)
    variants.append(("kitti_b3_f24_flospdepth_mono_2080ti infer_mode", recs, st))
    for what, recs, st in variants:
        sigs = {LR.signature(r, st) for r in recs}
        names |= {r[0] for r in recs}
        lines.append("%-40s %4d launches, %4d distinct, entry points %s"
                     % (what, len(recs), len(sigs), sorted({r[0] for r in recs})))
    with capsys.disabled():
        print("\nlaunch-replay census (tf32; non-convolution launches):\n" + "\n".join(lines)
              + "\n%d distinct launches over the six configurations' forward + class-map plans; %d entry points in all"
              % (total, len(names)))
    assert names <= set(LR.SPECS), names - set(LR.SPECS)
    assert names == set(LR.SPECS), set(LR.SPECS) - names
    for what, recs, st in variants:
        for r in recs:                      # every pointer lands in a storage the plan holds; every region fits
            LR.SPECS[r[0]].regions(LR.named(r), st)


# ---------------------------------------------------------------------------------------------------------------
# references against torch float64
def _g(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=f64)


def test_references_against_torch():
    x = _g(2, 9, 11, 16)
    w = _g(9, 16, seed=1)
    b = _g(16, seed=2)
    for K, S in ((3, 1), (3, 2)):
        OH, OW = -(-9 // S), -(-11 // S)
        ph, pw = max((OH - 1) * S + K - 9, 0), max((OW - 1) * S + K - 11, 0)
        out, v, _ = LR.dwconv_ref(x, w, b, K, S, ph // 2, pw // 2, OH, OW, "silu")
        xt = F.pad(x.permute(0, 3, 1, 2), [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2])
        want = F.conv2d(xt, w.t().reshape(16, 1, K, K), b, S, 0, 1, 16)
        assert torch.allclose(out, F.silu(want).permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    for OH, OW in ((13, 21), (1, 5)):
        r, _ = LR.bilinear_ac_ref(x, OH, OW)
        want = F.interpolate(x.permute(0, 3, 1, 2), size=(OH, OW), mode="bilinear", align_corners=True)
        assert torch.allclose(r, want.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    # the tapsum: nine shifted, zero-masked resizes
    ys = [_g(2, 4, 5, 8, seed=10 + t) for t in range(9)]
    pre = _g(2, 7, 9, 8, seed=3)
    out, _, _ = LR.tapsum_ref(ys, pre, 7, 9, "relu")
    want = pre.permute(0, 3, 1, 2).clone()
    for t, y in enumerate(ys):
        r = F.interpolate(y.permute(0, 3, 1, 2), size=(7, 9), mode="bilinear", align_corners=True)
        want += F.pad(r, [1, 1, 1, 1])[:, :, 1 + t // 3 - 1:8 + t // 3 - 1, 1 + t % 3 - 1:10 + t % 3 - 1]
    assert torch.allclose(out, F.relu(want).permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    z = _g(3, 7, 50)
    assert torch.allclose(LR.softmax_ref(z, 1), torch.softmax(z, 1), rtol=1e-12, atol=1e-15)
    pool = (_g(2, 24) * 2 ** 30).round().long()
    w1, b1, w2t, b2 = _g(6, 24, seed=4), _g(6, seed=5), _g(6, 24, seed=6), _g(24, seed=7)
    hidden, gate, _, _, _ = LR.se_mlp_ref(pool, 1 / 37, w1, b1, w2t, b2)
    mean = pool.double() / 2 ** 24 / 37
    h = F.silu(F.linear(mean, w1, b1))
    assert torch.allclose(hidden, h, rtol=1e-12) and torch.allclose(gate, torch.sigmoid(F.linear(h, w2t.t(), b2)))
    grid = torch.rand(1, 3, 4, 5, 3, generator=torch.Generator().manual_seed(8), dtype=f64) * 2.2 - 1.1
    depth = _g(2, 6, 7, 9).softmax(1)
    got, _ = LR.sample_mean(depth, [grid, grid], 0)
    want = sum(F.grid_sample(depth[v][None, None], grid, align_corners=False) for v in range(2))
    assert torch.allclose(got, want.reshape(-1), rtol=1e-12)


# ---------------------------------------------------------------------------------------------------------------
# the comparator: what it must accept and reject
def _resize_case(precision):
    ys = [_g(1, 5, 6, 8, seed=20 + t) for t in range(9)]
    pre = _g(1, 9, 11, 8, seed=30)
    out, v, S = LR.tapsum_ref(ys, pre, 9, 11, "none")
    o = LR.Out(ref=out, S=S, K=37, family="resize", store=precision, act="none", v=v)
    return ys, pre, o


def _rejects(got, o, precision):
    bad, _, _ = LR.check(got, o, precision)
    return bool(bad.any())


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_comparator_sharpness(precision):
    ys, pre, o = _resize_case(precision)
    q = LR.quantize(o.ref, precision)
    assert not _rejects(q, o, precision)
    # an fp32 reordering of the same sum, then rounded: accepted
    ys32 = [y.float() for y in ys]
    acc = pre.float().permute(0, 3, 1, 2).clone()
    for t, y in reversed(list(enumerate(ys32))):
        r = F.interpolate(y.permute(0, 3, 1, 2), size=(9, 11), mode="bilinear", align_corners=True)
        acc += F.pad(r, [1, 1, 1, 1])[:, :, t // 3:9 + t // 3, t % 3:11 + t % 3]
    assert not _rejects(LR.quantize(acc.permute(0, 2, 3, 1).double(), precision), o, precision)
    # truncation instead of rounding, and one ulp on one element
    assert _rejects(LR.quantize(o.ref, precision, "trunc"), o, precision)
    one = q.clone()
    at = (0, 4, 5, 3)
    one[at] += LR.ulp_store(one[at].abs(), precision) * torch.sign(one[at] - o.ref[at]).clamp(min=0).mul(2).sub(1)
    assert _rejects(one, o, precision)
    # a dropped border tap: tap (dy, dx) = (0, +1) missing in the last-but-one column
    r, _ = LR.bilinear_ac_ref(ys[5], 9, 11)
    dropped = q.clone()
    dropped[:, :, 9] = LR.quantize(o.ref[:, :, 9] - r[:, :, 10], precision)
    assert _rejects(dropped, o, precision)
    # a squeeze short by one block
    y = LR.quantize(_g(2, 20 * 40, 16, seed=40).relu(), precision)
    po = types.SimpleNamespace(B=2, C=16, OH=20, OW=40)
    full = (y.sum(1) * 2 ** 24).round().long()
    assert LR.check_pool(full, torch.zeros_like(full), y.reshape(-1, 16), po, precision)[0] == []
    short = full - (y[:, :8 * 16].sum(1) * 2 ** 24).round().long()
    assert LR.check_pool(short, torch.zeros_like(full), y.reshape(-1, 16), po, precision)[0]


def test_stray_store_and_dirty_pad_channels():
    """a store one channel window to the left, and pad channels written where the launch must not: the "nothing
    else moves" check on a copy_channels launch over CPU storages"""
    from occdepth_b200 import _lib
    src = torch.randn(10, 32)
    dst = torch.zeros(10, 40)
    st = LR.Storages([src, dst])
    rec = ("occd_copy_channels", [("p", src.data_ptr()), ("p", dst.data_ptr()), ("i", _lib.DTYPE_F32), ("l", 10),
                                  ("i", 8), ("i", 32), ("i", 8), ("i", 40), ("i", 16), ("s",)])
    L = LR.Launch(rec, st)
    before = L.snapshot()
    dst[:, 16:24] = src[:, 8:16]
    assert LR.moved(L, before) == []
    assert LR.compare(L, LR._ref_copy(L.a, [src[:, 8:16]], None, "tf32"),
                      [w.view(L.storages) for w in L.writes], "tf32")[0] == []
    dst[:, 8:16] = src[:, 8:16]                                  # one window to the left
    assert LR.moved(L, before)
    dst[:, 8:16] = 0
    dst[3, 24] = 1.0                                             # the channel after the window
    assert LR.moved(L, before)
