"""The occupied-voxel list on the device (occd_occupied_voxels, voxels.occupied_voxels, OccDepth.predict_voxels,
CameraPipeline(output="voxels")) against numpy's selection (oracle.voxel_list): every comparison is exact -- integers,
and float32 coordinates bit for bit."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import data as D
from occdepth_b200.voxels import HIST_BINS, occupied_voxels
from oracle import voxel_list as OV

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402

KITTI, NYU = (256, 256, 32), (60, 36, 60)


def _sc():
    import shipped_configs
    return shipped_configs


def _np(t):
    return t.cpu().numpy()


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _check(vl, maps, masks, voxel_size=None, origin=None, index0=0, what=""):
    """every frame of VoxelList `vl` against the oracle on the host arrays"""
    counts = vl.counts()
    for b, y in enumerate(maps):
        want = OV.voxel_list(y, None if masks is None else masks[b], voxel_size, origin, index0, HIST_BINS)
        n = int(want["count"].sum())
        assert counts[b].tolist() == want["count"].tolist(), (what, b)
        assert np.array_equal(_np(vl.hist[b]).astype(np.int64), want["hist"]), (what, b)
        w = min(n, vl.capacity)
        assert _same(_np(vl.index[b, :w]), want["index"][:w]), (what, b)
        assert _same(_np(vl.cls[b, :w]), want["cls"][:w]), (what, b)
        if voxel_size is not None:
            assert _same(_np(vl.xyz[b, :w]), want["xyz"][:w]), (what, b)
    return counts


def _random_map(shape, B, seed, kind):
    g = np.random.default_rng(seed)
    y = g.integers(1, 20, size=(B,) + tuple(shape)).astype(np.uint16)
    if kind == "sparse":
        y[g.random(y.shape) > 0.05] = 0
        y.reshape(-1)[g.integers(0, y.size, 100)] = 255
    elif kind == "skewed":                       # one dense block of one class, the rest empty
        y[:] = 0
        y[:, : shape[0] // 3, : shape[1] // 2] = 7
    elif kind == "empty":
        y[:] = 0
        y.reshape(-1)[::17] = 255
    elif kind == "one":
        y[:] = 0
        y.reshape(B, -1)[:, y[0].size // 2 + 3] = 5
    else:
        assert kind == "full"
    return y


# ---- 1. the kernel ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,res", [(KITTI, 0.2), (NYU, 0.08)])
@pytest.mark.parametrize("kind", ["sparse", "skewed", "empty", "full", "one"])
def test_list_equals_numpy(shape, res, kind):
    for B in (1, 2):
        y = _random_map(shape, B, 3 + B, kind)
        g = np.random.default_rng(9)
        n = y[0].size
        masks = {"none": None, "random": g.random((B, n)) < 0.4, "all_false": np.zeros((B, n), bool),
                 "all_true": np.ones((B, n), bool)}
        yd = torch.from_numpy(y).cuda()
        for name, m in masks.items():
            if B == 2 and name in ("all_false", "all_true"):
                continue
            origin = [0, -25.6, -2] if name == "random" else None
            vl = occupied_voxels(yd, m, voxel_size=res, vox_origin=origin)
            _check(vl, y, m, res, origin, what=(kind, B, name))
            assert not vl.truncated
            if kind == "empty":
                assert vl.counts().sum() == 0
            if name == "random" and B == 1:
                got = vl.rows()
                rows = OV.kitti_rows(y[0], m[0], res)
                for a, w in zip(got, rows):
                    w = w.copy()
                    w[:, :3] += np.asarray(origin, np.float64)
                    assert _same(a, OV.rows32(w))
        # without coordinates, and twice: identical bytes
        m = masks["random"]
        a = occupied_voxels(yd, m)
        b = occupied_voxels(yd, m)
        assert a.xyz is None
        _check(a, y, m, what=(kind, B, "no xyz"))
        for k in ("count", "hist", "index", "cls"):
            na = int(a.counts()[0].sum())
            assert torch.equal(getattr(a, k)[0, :na].view(torch.uint8), getattr(b, k)[0, :na].view(torch.uint8)), k


def test_odd_sizes_misaligned_views_and_remapped_ids():
    g = np.random.default_rng(0)
    for shape in ((7, 5, 3), (13, 11, 9), (3, 683, 1), (1, 1, 1), (17, 16, 8)):
        n = int(np.prod(shape))
        for B, off in ((1, 0), (2, 0), (2, 1), (3, 5)):
            y = g.integers(0, 100, size=(B,) + shape).astype(np.uint16)       # ids above the histogram's 64 bins
            y[g.random(y.shape) < 0.5] = 0
            y.reshape(-1)[g.integers(0, y.size, 3)] = 255
            m = g.random((B, n)) < 0.5
            big = torch.zeros(off + B * n + 8, dtype=torch.uint16, device="cuda")
            big[off:off + B * n] = torch.from_numpy(y.reshape(-1)).cuda()
            yd = big[off:off + B * n].view((B,) + shape)
            mb = torch.zeros(off + B * n + 8, dtype=torch.bool, device="cuda")
            mb[off:off + B * n] = torch.from_numpy(m.reshape(-1)).cuda()
            vl = occupied_voxels(yd, mb[off:off + B * n], voxel_size=0.08, index0=7 * shape[1] * shape[2])
            _check(vl, y, m, 0.08, None, 7 * shape[1] * shape[2], what=(shape, B, off))
            assert int(vl.hist.sum()) == int(((y > 0) & (y < 64)).sum())


def test_truncation_keeps_order_counts_and_the_bytes_past_capacity():
    y = _random_map(KITTI, 2, 1, "sparse")
    m = np.random.default_rng(2).random((2, y[0].size)) < 0.4
    yd = torch.from_numpy(y).cuda()
    full = occupied_voxels(yd, m, voxel_size=0.2)
    total = full.counts().sum(1)
    n_in = int(full.counts()[0, 0])
    for cap in (0, 1, n_in - 3, n_in + 5, int(total.min()), int(total.max()) + 9):
        out = occupied_voxels(yd, m, voxel_size=0.2, capacity=cap)       # allocate, then fill with a canary
        out.index.fill_(-7)
        out.cls.view(torch.int16).fill_(-7)
        out.xyz.fill_(-7.0)
        vl = occupied_voxels(yd, m, voxel_size=0.2, capacity=cap, out=out)
        assert vl is out
        _check(vl, y, m, 0.2, what=cap)
        assert vl.truncated == bool((total > cap).any())
        for b in range(2):
            w = min(cap, int(total[b]))
            assert bool((vl.index[b, w:] == -7).all()) and bool((vl.cls[b, w:].view(torch.int16) == -7).all())
            assert bool((vl.xyz[b, w:] == -7.0).all())
            ni, no, first_out = vl.split(b)
            assert ni + no == w
        if 0 < cap < n_in:
            assert vl.rows(0)[1].shape == (0, 4) and vl.rows(0)[0].shape == (cap, 4)
    with pytest.raises(ValueError, match="another shape"):
        occupied_voxels(yd, m, voxel_size=0.2, capacity=5, out=full)


def test_refusals():
    y = torch.zeros(1, 4, 4, 4, dtype=torch.uint16, device="cuda")
    with pytest.raises(TypeError):
        occupied_voxels(y.cpu())
    with pytest.raises(TypeError):
        occupied_voxels(torch.zeros(1, 4, 4, 4, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        occupied_voxels(y, np.zeros(63, bool))
    with pytest.raises(TypeError):
        occupied_voxels(y, np.zeros(64, np.float32))
    with pytest.raises(ValueError):
        occupied_voxels(y, vox_origin=[0, 0, 0])
    with pytest.raises(ValueError):
        occupied_voxels(y.expand(2, 4, 4, 4)[:, :, ::2])
    with pytest.raises(ValueError, match="no coordinates"):
        occupied_voxels(y).rows()


# ---- 2. the model ----------------------------------------------------------------------------------------------------
def _count_builds(m, monkeypatch):
    n = [0]
    orig = m._build

    def counted(*a, **k):
        n[0] += 1
        return orig(*a, **k)
    monkeypatch.setattr(m, "_build", counted)
    return n


def _with_fov_mask_1(m, batch, seed=5):
    """the batch with the `fov_mask_1` the datasets add: bool (V, N1, P) per frame at the output resolution"""
    if "fov_mask_1" in batch:
        return batch
    V = batch["img"].shape[1]
    n1 = int(np.prod(m.full_scene_size))
    g = torch.Generator().manual_seed(seed)
    return dict(batch, fov_mask_1=[(torch.rand(V, n1, 1, generator=g) < 0.4).cuda()])


CASES = [(n, "tf32") for n in _sc().CONFIGS] + [("nyu_b4_f100_2080ti", "bf16"), ("kitti_b3_f32_flospdepth_2080ti", "bf16")]


@pytest.mark.parametrize("name,precision", CASES)
def test_shipped_config_predict_voxels(name, precision, monkeypatch):
    sc = _sc()
    gc.collect()
    torch.cuda.empty_cache()
    m, batch, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    batch = _with_fov_mask_1(m, sc.to_cuda(batch))
    res = 0.08 if m.dataset == "NYU" else 0.2
    nyu = m.dataset == "NYU"                      # NYU lists every occupied voxel as inside, as its script does
    mask = None if nyu else _np(batch["fov_mask_1"][0][0, :, 0])
    masks = None if nyu else [mask]
    inv = np.random.default_rng(3).permutation(np.arange(1, 250))[:m.n_classes]
    inv[0] = 0
    with torch.no_grad():
        y = _np(m.predict_classes(batch))
        builds = _count_builds(m, monkeypatch)
        vl = m.predict_voxels(batch)
        c = _check(vl, y, masks, res, what=name)
        assert c.sum() > 0 and vl.capacity == y[0].size and (c[0, 1] > 0) == (not nyu)
        m.predict_classes(batch)
        vl = m.predict_voxels(batch, fov_mask=False, capacity=1000)
        _check(vl, y, None, res, what=(name, "no mask"))
        assert builds[0] == 0
        y_inv = _np(m.predict_classes(batch, inv))
        _check(m.predict_voxels(batch, inv_map=inv, vox_origin=[0, -25.6, -2]), y_inv, masks, res, [0, -25.6, -2],
               what=(name, "inv_map"))
    del m
    gc.collect()
    torch.cuda.empty_cache()


def _host_fov_mask_1(m, frame, geo):
    """the mask the reference's host vox2pix gives at scale 1 for the first view's centre pixel (KITTI)"""
    from oracle.projection import vox2pix
    H, W = geo["img_hw"]
    return vox2pix(frame["T_velo_2_cam"][0], frame["cam_k"][0], geo["vox_origin"], geo["voxel_size"] / m.project_scale,
                   W, H, geo["scene_size"], 0)[1][:, 0]


@pytest.mark.parametrize("dataset", ["kitti", "NYU"])
def test_camera_frames_and_pipeline(dataset, monkeypatch):
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    if dataset == "NYU":
        m, _, _ = sc.make_case("nyu_b4_f100_2080ti")
        geo = dict(img_hw=sc.NYU_IMG)
        frames = [nyu_frame(1), nyu_frame(2), nyu_frame(3)]
        frames[1]["cam_pose"][0, 3] += 0.2
        res, want_calls = 0.08, [2, 2, 2, 2]     # a new pose every frame: two views' indices; NYU takes no mask
    else:
        hw, full = (96, 320), (64, 64, 16)
        m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
        geo = kitti_geometry(hw[0], hw[1], full)
        frames = [kitti_frame(2, hw[0], hw[1], 10), kitti_frame(2, hw[0], hw[1], 11),
                  kitti_frame(2, hw[0], hw[1], 12, shift=0.3)]
        res, want_calls = 0.2, [3, 0, 3, 3]      # two views' indices and the mask; one calibration serves frames 0 and 1; the last frame is frame 0 again
    m = m.cuda().set_precision("bf16")
    calls = []
    orig = D.vox2pix_into
    monkeypatch.setattr(D, "vox2pix_into", lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
    seq = frames + frames[:1]
    with torch.no_grad():
        want_y = [_np(m.predict_frame(dict(f, **geo))) for f in seq]
        masks = [None if dataset == "NYU" else _host_fov_mask_1(m, f, geo) for f in seq]
        m.invalidate_plans()
        lists = []
        for i, f in enumerate(seq):
            n0 = len(calls)
            vl = m.predict_voxels(dict(f, **geo))
            assert len(calls) - n0 == want_calls[i], (i, len(calls) - n0)
            c = _check(vl, want_y[i], None if masks[i] is None else [masks[i]], res, what=(dataset, i))
            assert c[0, 0] > 0 and (c[0, 1] > 0) == (dataset == "kitti")
            lists.append(OV.voxel_list(want_y[i][0], masks[i], res))
        # the pipeline: the same lists per ticket, one of them truncated
        cap = max(int(w["count"].sum()) for w in lists) - 1            # the fullest frame loses its last row
        pipe = CameraPipeline(m, output="voxels", capacity=cap, **geo)
        got = {}

        def keep(t):
            r = pipe.result(t)
            got[t] = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in r.items()}
        for f in seq:
            t = pipe.submit(f)
            if t is not None:
                keep(t)
        keep(pipe.flush())
    assert any(g["truncated"] for g in got.values())
    for i, w in enumerate(lists):
        g = got[i]
        n = min(cap, int(w["count"].sum()))
        assert g["count"].tolist() == w["count"].tolist() and g["truncated"] == (int(w["count"].sum()) > cap)
        assert np.array_equal(g["hist"].astype(np.int64), w["hist"])
        for k in ("index", "cls", "xyz"):
            assert _same(g[k], w[k][:n]), (i, k)
    assert pipe.d2h_bytes == 4 * (2 + HIST_BINS) + cap * (4 + 2 + 12)
    del m, pipe
    gc.collect()
    torch.cuda.empty_cache()


# ---- 3. the X-slab partition ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [2, 3])
def test_slab_lists_concatenate(R, monkeypatch):
    from occdepth_b200.parallel import SimSlabGroup
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    gc.collect()
    torch.cuda.empty_cache()
    m, batch, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti")
    m = m.cuda().set_precision("bf16")
    batch = _with_fov_mask_1(m, sc.to_cuda(batch))
    mask = _np(batch["fov_mask_1"][0][0, :, 0])
    with torch.no_grad():
        y = _np(m.predict_classes(batch))
    want = OV.voxel_list(y[0], mask, 0.2)
    m.invalidate_plans()
    # the R rank plans in lock-step on one device, as tests/test_gpu_class_map.py runs them; then every rank lists its
    # slab as predict_voxels does under enable_slab_parallel (the plan's x_range, the batch's whole mask)
    img = batch["img"]
    B, V, _, H, W = img.shape
    pp, fm = batch["projected_pix_2"], batch["fov_mask_2"]
    N, P = pp[0].shape[1], pp[0].shape[2]
    grp = SimSlabGroup(R, halo=3)
    ents = []
    try:
        for r in range(R):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                ents.append(m._build(B, V, H, W, N, P, img.device, batch, classes=("classes", None)))
    finally:
        m.__dict__.pop("slab_ctx", None)
        m.invalidate_plans()
    for e in ents:
        m._stage(e, batch, img, pp, fm, img.device)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
        parts = [m._list_voxels(e[4], e[0].x_range, batch["fov_mask_1"], None, None, None, None) for e in ents]
    assert [e[0].x_range[0] for e in ents][0] == 0 and ents[-1][0].x_range[1] == 256
    n_in = [int(p.counts()[0, 0]) for p in parts]
    n_all = [int(p.counts()[0].sum()) for p in parts]
    assert sum(n_all) == int(want["count"].sum()) and sum(n_in) == int(want["count"][0])
    for k in ("index", "cls", "xyz"):
        cat = np.concatenate([_np(getattr(p, k)[0, :n]) for p, n in zip(parts, n_in)] +
                             [_np(getattr(p, k)[0, n:t]) for p, n, t in zip(parts, n_in, n_all)])
        assert _same(cat, want[k]), k
    del m
    gc.collect()
    torch.cuda.empty_cache()
