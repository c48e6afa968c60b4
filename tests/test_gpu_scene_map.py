"""Scene maps on the device (occd_scene_map_integrate / _shift / _mark_unobserved, fusion.SceneMap,
OccDepth.fuse_frames) against the numpy restatement in oracle/scene_map.py, against predict_frame, and across the
Python and model-file routes."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from occdepth_b200.fusion import SceneMap
from occdepth_b200.models.OccDepth import OccDepth
from occdepth_b200.voxels import occupied_voxels
from oracle import scene_map as ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def rigid(yaw, t):
    T = np.eye(4)
    T[:2, :2] = [[np.cos(yaw), -np.sin(yaw)], [np.sin(yaw), np.cos(yaw)]]
    T[:3, 3] = t
    return T


def random_probs(C, storage, seed):
    """float16 softmax-like probabilities with exact zeros and NaN-poisoned voxels"""
    g = np.random.default_rng(seed)
    x = g.standard_normal((C,) + storage) * 2
    p = np.exp(x) / np.exp(x).sum(0, keepdims=True)
    p[g.random(p.shape) < 0.05] = 0.0
    plane = p.reshape(C, -1)
    bad = g.choice(plane.shape[1], plane.shape[1] // 50, replace=False)
    plane[g.integers(0, C, bad.size), bad] = np.nan
    return p.astype(np.float16)


def _tol(want, term):
    """the per-frame bound of the fp32 accumulation: device logf and numpy log each within an ulp or so"""
    return 4 * np.spacing(np.maximum(np.abs(want), np.abs(term)).astype(np.float32))


SEQ = [  # (pose, axes, with mask)
    (np.eye(4), "xyz", False),
    (rigid(np.pi / 6, (1.3, -0.7, 0.1)), "xyz", True),
    (rigid(-np.pi / 2, (5.0, 2.0, -0.3)), "xzy", True),
    (rigid(np.pi, (14.0, 3.0, 0.0)), "xzy", False),      # partly outside the map
]


def _frame(i, C=20):
    axes = SEQ[i][1]
    storage = (40, 32, 8) if axes == "xyz" else (40, 8, 32)
    p = random_probs(C, storage, 10 + i)
    mask = None
    if SEQ[i][2]:
        mask = np.random.default_rng(50 + i).random(storage) < 0.7
    return p, mask


GRID_ORIGIN, GRID_VOXEL = np.array([0.0, -3.2, -0.8]), 0.2
MAP = dict(dims=(80, 72, 12), voxel=0.2, origin=(-3.0, -7.0, -1.2))


def _integrate(smap, i, C=20):
    p, mask = _frame(i, C)
    pose, axes, _ = SEQ[i]
    m = None if mask is None else torch.from_numpy(mask).cuda()
    smap.integrate(torch.from_numpy(p).cuda(), pose, GRID_ORIGIN, GRID_VOXEL, axes=axes, fov_mask=m)
    return p, mask


def test_integrate_matches_the_oracle():
    C = 20
    smap = SceneMap(C, MAP["dims"], MAP["voxel"], MAP["origin"])
    acc_ref = np.zeros((C,) + MAP["dims"], np.float32)
    cnt_ref = np.zeros(MAP["dims"], np.int32)
    worst = 0.0
    for i in range(len(SEQ)):
        before = smap.acc.cpu().numpy().copy()
        cnt_before = smap.count.cpu().numpy().copy()
        p, mask = _integrate(smap, i)
        torch.cuda.synchronize()
        acc, cnt = smap.acc.cpu().numpy(), smap.count.cpu().numpy()
        # the oracle's step from the device's own previous state, and the whole sequence in the oracle alone
        step = before.copy()
        cstep = cnt_before.copy()
        obs = ref.integrate(step, cstep, MAP["origin"], MAP["voxel"], p, SEQ[i][0], GRID_ORIGIN, GRID_VOXEL,
                            SEQ[i][1], mask)
        ref.integrate(acc_ref, cnt_ref, MAP["origin"], MAP["voxel"], p, SEQ[i][0], GRID_ORIGIN, GRID_VOXEL,
                      SEQ[i][1], mask)
        assert 0 < int(obs.sum()) < obs.size, i
        assert np.array_equal(cnt, cstep), i                                   # the written set and the counts
        assert np.array_equal(cnt, cnt_ref), i
        assert acc[:, ~obs].tobytes() == before[:, ~obs].tobytes(), i          # nothing else moved
        term = step[:, obs] - before[:, obs]
        d = np.abs(acc[:, obs] - step[:, obs])
        assert (d <= _tol(step[:, obs], term)).all(), (i, float(d.max()))
        worst = max(worst, float((d / np.spacing(np.abs(step[:, obs]) + 1e-30)).max()))
    print("largest per-frame difference: %.1f ulp" % worst)
    # the arg-max of the map where the oracle's top two are further apart than the accumulated bound
    cmap = smap.classes().cpu().numpy()
    srt = np.sort(acc_ref, 0)
    gap = srt[-1] - srt[-2]
    clear = (cnt_ref > 0) & (gap > len(SEQ) * 4 * np.spacing(np.abs(srt[-1]).astype(np.float32)))
    assert np.array_equal(cmap[clear], np.argmax(acc_ref, 0)[clear])
    assert (cmap[cnt_ref == 0] == 255).all()


def test_two_maps_hold_the_same_bytes():
    maps = [SceneMap(20, MAP["dims"], MAP["voxel"], MAP["origin"]) for _ in range(2)]
    for smap in maps:
        for i in range(len(SEQ)):
            _integrate(smap, i)
    assert _same(maps[0].acc, maps[1].acc) and _same(maps[0].count, maps[1].count)
    maps[0].reset()
    assert not maps[0].acc.any() and not maps[0].count.any()


def test_shift():
    smap = SceneMap(20, MAP["dims"], MAP["voxel"], MAP["origin"])
    _integrate(smap, 0)
    _integrate(smap, 1)
    for d in [(3, -2, 1), (-5, 0, 0), (0, 7, -2), (200, 0, 0)]:
        acc0, cnt0 = smap.acc.cpu().numpy(), smap.count.cpu().numpy()
        o0 = smap.origin.copy()
        smap.shift(d)
        assert np.array_equal(smap.acc.cpu().numpy(), ref.shift(acc0, d))
        assert np.array_equal(smap.count.cpu().numpy(), ref.shift(cnt0, d))
        assert np.array_equal(smap.origin, o0 + np.asarray(d, np.float64) * smap.voxel)
        if d[0] == 200:
            assert not smap.count.any()
    # integrating after shift(d) is integrating into a map built at the shifted origin with the shifted contents
    a = SceneMap(20, MAP["dims"], MAP["voxel"], MAP["origin"])
    _integrate(a, 0)
    acc0, cnt0 = a.acc.cpu().numpy(), a.count.cpu().numpy()
    a.shift((4, -3, 1))
    b = SceneMap(20, MAP["dims"], MAP["voxel"], a.origin)
    b.acc.copy_(torch.from_numpy(ref.shift(acc0, (4, -3, 1))))
    b.count.copy_(torch.from_numpy(ref.shift(cnt0, (4, -3, 1))))
    _integrate(a, 1)
    _integrate(b, 1)
    assert _same(a.acc, b.acc) and _same(a.count, b.count)


def test_queries_reuse_the_class_map_kernels():
    C = 20
    smap = SceneMap(C, MAP["dims"], MAP["voxel"], MAP["origin"])
    _integrate(smap, 0)
    _integrate(smap, 1)
    unobs = smap.count == 0
    assert bool(unobs.any()) and not bool(unobs.all())
    inv = np.random.default_rng(3).permutation(250)[:C]
    for kw in (dict(), dict(inv_map=inv, unknown=300)):
        want = OccDepth.class_map(smap.acc[None], kw.get("inv_map"))[0]
        want = torch.where(unobs, torch.tensor(kw.get("unknown", 255), dtype=torch.int32, device="cuda"),
                           want.int()).to(torch.uint16)
        got = smap.classes(**kw)
        assert _same(got, want)
        wm, wc = OccDepth.class_map(smap.acc[None], kw.get("inv_map"), confidence=True)
        gm, gc = smap.classes(confidence=True, **kw)
        assert _same(gm, want) and _same(gc, wc[0])
        wm, wp = OccDepth.class_map(smap.acc[None], kw.get("inv_map"), probabilities=True)
        gm, gp = smap.classes(probabilities=True, **kw)
        assert _same(gm, want) and _same(gp, wp[0])
        assert float((gc[unobs].float() - 1.0 / C).abs().max()) <= 5e-5          # softmax of zeros
        vl = smap.voxels(**kw)
        wl = occupied_voxels(want, voxel_size=smap.voxel, vox_origin=smap.origin, ignore=kw.get("unknown", 255))
        assert np.array_equal(vl.counts(), wl.counts())
        r, w = vl.rows(), wl.rows()
        assert all(np.array_equal(x, y) for x, y in zip(r, w)) and r[0].shape[0] > 0


# ---- models ----------------------------------------------------------------------------------------------------------
KITTI_IMG, KITTI_FULL = (96, 320), (64, 64, 16)


def _kitti_model(precision="tf32"):
    import shipped_configs
    m, _, _ = shipped_configs.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=KITTI_IMG, full=KITTI_FULL)
    return m.cuda().set_precision(precision)


def _kitti_frames(n):
    H, W = KITTI_IMG
    geo = kitti_geometry(H, W, KITTI_FULL)
    return [dict(kitti_frame(2, H, W, 1 + i, shift=0.3 * i), **geo) for i in range(n)]


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_identity_fusion_is_predict_frame(precision):
    _free()
    m = _kitti_model(precision)
    f = _kitti_frames(1)[0]
    with torch.no_grad():
        cmap, probs = m.predict_frame(f, probabilities=True)
        smap = SceneMap(m.n_classes, KITTI_FULL, 0.2, f["vox_origin"])
        assert m.fuse_frames(smap, f, np.eye(4)) is smap
        fov = m._frame_fov_mask_1(m._frame_inputs(f, torch.device("cuda"))).view(KITTI_FULL)
        got = smap.classes().int()
    assert torch.equal(smap.count == 0, ~fov)
    assert bool((got[~fov] == 255).all())
    diff = fov & (got != cmap[0].int())
    p = probs[0].float()
    top2 = p.topk(2, dim=0).values
    ties = diff & (top2[0] == top2[1])
    assert torch.equal(diff, ties), int((diff & ~ties).sum())
    # at a tie the map holds the first of the float16 maxima
    assert torch.equal(got[diff].long(), p.argmax(0)[diff])
    print("%s: %d of %d observed voxels differ from predict_frame, each at a float16 tie"
          % (precision, int(diff.sum()), int(fov.sum())))
    del m
    _free()


def test_fuse_frames_list_and_model_file(tmp_path):
    from occdepth_b200 import deploy
    _free()
    m = _kitti_model()
    frames = _kitti_frames(3)
    poses = [rigid(0.05 * i, (0.6 * i, 0.2 * i, 0.0)) for i in range(3)]
    geo = dict(dims=(96, 80, 16), voxel=0.2, origin=(-1.0, -8.0, -2.0))
    with torch.no_grad():
        a = SceneMap(m.n_classes, geo["dims"], geo["voxel"], geo["origin"])
        m.fuse_frames(a, frames, poses)
        b = SceneMap(m.n_classes, geo["dims"], geo["voxel"], geo["origin"])
        _, probs = m.predict_frames(frames, probabilities=True)
        for i, f in enumerate(frames):
            fi = m._frame_inputs(f, torch.device("cuda"))
            b.integrate(probs[i], poses[i], f["vox_origin"], 0.2, fov_mask=m._frame_fov_mask_1(fi, None, i))
        assert _same(a.acc, b.acc) and _same(a.count, b.count)
        assert int((a.count == 3).sum()) > 0
        deploy.export(m, tmp_path / "probs.occd", frames, probabilities=True)
    lm = deploy.LoadedModel(tmp_path / "probs.occd")
    _, fprobs = lm.run_frames(frames, probs=True)
    c = SceneMap(m.n_classes, geo["dims"], geo["voxel"], geo["origin"])
    for i, f in enumerate(frames):
        fi = m._frame_inputs(f, torch.device("cuda"))
        c.integrate(fprobs[i], poses[i], f["vox_origin"], 0.2, fov_mask=m._frame_fov_mask_1(fi, None, i))
    lm.close()
    assert _same(a.acc, c.acc) and _same(a.count, c.count)
    del m, lm
    _free()


def test_fuse_frames_nyu():
    import shipped_configs
    _free()
    m, _, _ = shipped_configs.make_case("nyu_b4_f100_2080ti")
    m = m.cuda().set_precision("tf32")
    f = dict(nyu_frame(1), img_hw=shipped_configs.NYU_IMG)
    pose = rigid(0.3, (0.2, -0.1, 0.0))                      # map <- world
    with torch.no_grad():
        a = SceneMap(m.n_classes, (70, 70, 40), 0.08, (-2.5, 0.0, -0.3))
        m.fuse_frames(a, [f], [pose])
        _, probs = m.predict_frames([f], probabilities=True)
        b = SceneMap(m.n_classes, (70, 70, 40), 0.08, (-2.5, 0.0, -0.3))
        b.integrate(probs[0], pose, f["vox_origin"], 0.08, axes="xzy")
    assert _same(a.acc, b.acc) and _same(a.count, b.count)
    assert int((a.count > 0).sum()) > 0
    del m
    _free()
