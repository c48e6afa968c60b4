"""Camera frames in, class map out (OccDepth.predict_frame, serving.CameraPipeline): the staging kernels against the
library's own two-step route, and every shipped configuration against the batch the reference's host route builds
(numpy normalisation, the numpy restatement of vox2pix, load_depth, the collate layout), bit for bit."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _lib
from occdepth_b200 import data as D
from occdepth_b200.engine import CL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import host_batch, kitti_frame, kitti_geometry, nyu_frame  # noqa: E402


def _sc():
    import shipped_configs
    return shipped_configs


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


# ---- 1. the staging kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_stage_rgb_equals_normalize_then_planar_to_cl(precision):
    dt = {"tf32": _lib.DTYPE_F32, "bf16": _lib.DTYPE_BF16}[precision]
    g = torch.Generator(device="cuda").manual_seed(0)
    # (raw H0, W0, crop H, W, row stride, image stride) in bytes: dense, odd W with a crop, padded rows and a gap
    for H0, W0, H, W, rs, ist in ((24, 40, 24, 40, 120, 2880), (37, 53, 30, 41, 170, 7000),
                                  (21, 33, 19, 31, 112, 2500)):
        buf = torch.randint(0, 256, (2 * ist,), dtype=torch.uint8, device="cuda", generator=g)
        imgs = torch.as_strided(buf, (2, H0, W0, 3), (ist, rs, 3, 1))
        out = torch.full((2, 1, H, W, 8), float("nan"), device="cuda",
                         dtype=torch.float32 if dt == _lib.DTYPE_F32 else torch.bfloat16)
        D.stage_rgb_u8(imgs, out, dt, H, W)
        for i in range(2):
            ref = CL.from_planar(D.normalize_rgb(imgs[i].contiguous(), H, W).unsqueeze(0), precision=precision)
            assert torch.equal(_bits(out[i:i + 1]), _bits(ref.buf)), (H0, W0, H, W, i)
            assert not torch.any(_bits(out[i, ..., 3:]) != 0)           # pad channels written as zeros


def test_stage_rgb_refuses_bad_args():
    img = torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda")
    out = torch.zeros(1, 1, 8, 8, 8, device="cuda")
    with pytest.raises(RuntimeError):
        D.stage_rgb_u8(img, torch.zeros(1, 1, 9, 9, 8, device="cuda"), _lib.DTYPE_F32, 9, 9)   # crop outside
    with pytest.raises(ValueError):
        D.stage_rgb_u8(img, out.bfloat16(), _lib.DTYPE_F32, 8, 8)                            # wrong out type


def test_depth_u16_to_f32_every_value():
    u = torch.arange(65536, dtype=torch.int32).to(torch.uint16)
    for divisor in (8000.0, 3000.0):
        out = torch.full((65536,), float("nan"), device="cuda")
        D.depth_u16_to_f32(u.cuda(), out, divisor, 10.0)
        want = (u.numpy() / divisor).astype("float32")
        want[want > 10] = 10
        want[want < 0] = 0
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), divisor


def _u16_equal(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _count_builds(m, monkeypatch):
    n = [0]
    orig = m._build

    def counted(*a, **k):
        n[0] += 1
        return orig(*a, **k)
    monkeypatch.setattr(m, "_build", counted)
    return n


# ---- 2. every shipped configuration ---------------------------------------------------------------------------------
CASES = [(n, "tf32") for n in _sc().CONFIGS] + [("nyu_b4_f100_2080ti", "bf16"), ("kitti_b3_f32_flospdepth_2080ti", "bf16")]


@pytest.mark.parametrize("name,precision", CASES)
def test_shipped_config_frame_parity(name, precision, monkeypatch):
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    gc.collect()
    torch.cuda.empty_cache()
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    spec = sc.CONFIGS[name]
    if spec["dataset"] == "NYU":
        geo = dict(img_hw=sc.NYU_IMG)
        frames = [nyu_frame(1), nyu_frame(2)]
        frames[1]["cam_pose"][0, 3] += 0.2
    else:
        H, W = sc.KITTI_IMG
        geo = kitti_geometry(H, W, sc.KITTI_FULL)
        frames = [kitti_frame(spec["views"], H, W, 1), kitti_frame(spec["views"], H, W, 2)]
    batches = [host_batch(m, f, geo) for f in frames]
    inv = np.random.default_rng(3).permutation(256)[:m.n_classes]
    with torch.no_grad():
        want = [m.predict_classes(b) for b in batches]
        want_inv = m.predict_classes(batches[0], inv)
        want_logits = m(batches[0])["ssc_logit"]
        builds = _count_builds(m, monkeypatch)
        f0 = dict(frames[0], **geo)
        assert _u16_equal(m.predict_frame(f0, inv_map=inv), want_inv)
        got = m.predict_frame(f0)
        assert _u16_equal(got, want[0]), int((got.int() != want[0].int()).sum())
        logits = m.predict_frame(f0, classes=False)["ssc_logit"]
        assert torch.equal(_bits(logits), _bits(want_logits))
        # one rebuild: the class-map cache holds one plan, and the remapped one had evicted the plain one; the frame
        # reused the tensor batch's remapped and forward plans as they were
        assert builds[0] == 1
        pipe = CameraPipeline(m, classes=True, **geo)
        got = {}
        for f in frames + frames[:1]:
            t = pipe.submit(f)
            if t is not None:
                r = pipe.result(t)
                assert r.is_pinned()
                got[t] = r.clone()
        got[pipe.flush()] = pipe.result(pipe.flush()).clone()
    for i, w in enumerate(want + want[:1]):
        assert got[i].dtype == torch.uint16 and _u16_equal(got[i], w.cpu()), i
    del m, pipe
    gc.collect()
    torch.cuda.empty_cache()


# ---- 3. the calibration cache ---------------------------------------------------------------------------------------
def test_calibration_cache(monkeypatch):
    import synthetic
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, other, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    m = m.cuda().set_precision("bf16")
    geo = kitti_geometry(hw[0], hw[1], full)
    frames = [kitti_frame(2, hw[0], hw[1], 10 + i) for i in range(6)]
    frames.append(kitti_frame(2, hw[0], hw[1], 16, shift=0.3))     # a changed T_velo_2_cam
    want = [m.predict_classes(host_batch(m, f, geo)) for f in frames]
    other = sc.to_cuda(other)
    N = other["projected_pix_2"][0].shape[1]
    pix, fov = synthetic.random_indices(N, hw[1], hw[0], n_views=2, seed=7)
    other.update(projected_pix_2=[pix.cuda()], fov_mask_2=[fov.cuda()])
    calls = []
    orig = D.vox2pix_into
    monkeypatch.setattr(D, "vox2pix_into", lambda *a, **k: (calls.append(1), orig(*a, **k))[1])
    per_frame = []
    with torch.no_grad():
        for i, f in enumerate(frames):
            if i == 3:
                m.predict_classes(other)           # overwrites the plan's index buffers
            n0 = len(calls)
            got = m.predict_frame(dict(f, **geo))
            per_frame.append(len(calls) - n0)
            assert _u16_equal(got, want[i]), i
    assert per_frame == [2, 0, 0, 2, 0, 0, 2]


# ---- 4. refusals ----------------------------------------------------------------------------------------------------
def test_refusals():
    from occdepth_b200.parallel import SimSlabGroup
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    geo = kitti_geometry(hw[0], hw[1], full)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    m = m.cuda()
    f = kitti_frame(2, hw[0], hw[1], 0)
    two = dict(f, img=np.stack([f["img"]] * 2), **geo)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="one frame"):
            m.predict_frame(two)
        pipe = CameraPipeline(m, **geo)
        with pytest.raises(NotImplementedError, match="one frame"):
            pipe.submit(two)
        for _ in range(3):
            t = pipe.submit(f)
        assert t == 1
        pipe.result(t)
        with pytest.raises(ValueError):
            pipe.result(0)                         # its buffer has been reused
        with pytest.raises(ValueError):
            pipe.result(3)
        m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        try:
            with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
                m.predict_frame(dict(f, **geo))
            with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
                CameraPipeline(m, **geo)
        finally:
            m.__dict__.pop("slab_ctx", None)
    mi, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full, infer_mode=True)
    mi = mi.cuda()
    with pytest.raises(NotImplementedError, match="infer_mode"):
        mi.predict_frame(dict(f, **geo))
    with pytest.raises(NotImplementedError, match="infer_mode"):
        CameraPipeline(mi, **geo)
