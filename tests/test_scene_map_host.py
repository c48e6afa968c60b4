"""Scene maps without a device: the kernel's index function (csrc/scene_map.cuh, run on the CPU by
tests/host_emul/scene_map_emul.cu) against the float64 numpy restatement (oracle/scene_map.py) bit for bit, the
launch box against brute force, and the refusals of the three entry points, SceneMap and OccDepth.fuse_frames."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, fusion
from oracle import scene_map as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("smap_emul") / "libsmap_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "scene_map_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).scene_map_index_emulate
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_double,
                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def run_emul(fn, T, origin, voxel, dims, grid_origin, grid_voxel, G, s):
    R = np.ascontiguousarray(np.linalg.inv(np.asarray(T, np.float64))[:3])
    o = np.ascontiguousarray(origin, np.float64)
    g = np.ascontiguousarray(grid_origin, np.float64)
    Ga = np.ascontiguousarray(G, np.int32)
    sa = np.ascontiguousarray(s, np.int64)
    n = int(np.prod(dims))
    off = np.full(n, -7, np.int64)
    f = np.full((n, 3), np.nan)
    assert fn(R.ctypes.data, o.ctypes.data, float(voxel), *dims, g.ctypes.data, float(grid_voxel), Ga.ctypes.data,
              sa.ctypes.data, off.ctypes.data, f.ctypes.data) == 0
    return off.reshape(dims), f.reshape(tuple(dims) + (3,))


def rigid(yaw, t, pitch=0.0, roll=0.0):
    cz, sz, cy, sy, cx, sx = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch), np.cos(roll), np.sin(roll)
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T


def _cases():
    rng = np.random.default_rng(5)
    out = [("identity", np.eye(4), (0.0, 0.0, 0.0), 0.2, (0.0, 0.0, 0.0), 0.2, "xyz"),
           ("yaw90", rigid(np.pi / 2, (3.0, -1.0, 0.2)), None, 0.2, (0.0, -2.0, -1.0), 0.4, "xyz"),
           ("yaw180", rigid(np.pi, (1.0, 2.0, 0.0)), None, 0.25, (-1.0, -1.0, -0.5), 0.2, "xzy"),
           # map centres (i + 0.5) * 0.4 + 0 and frame faces 0.2 + f * 0.4: every centre lies exactly on a face
           ("faces", np.eye(4), (0.0, 0.0, 0.0), 0.4, (0.2, 0.2, 0.2), 0.4, "xyz"),
           ("faces_xzy", np.eye(4), (0.0, 0.0, 0.0), 0.2, (0.1, -0.3, 0.1), 0.2, "xzy")]
    for i in range(4):
        T = rigid(rng.uniform(-np.pi, np.pi), rng.uniform(-2, 2, 3), rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3))
        out.append(("random%d" % i, T, None, rng.uniform(0.15, 0.3), tuple(rng.uniform(-1, 1, 3)),
                    rng.uniform(0.15, 0.4), "xyz" if i % 2 else "xzy"))
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_index_function_matches_the_oracle_bit_for_bit(emul, case):
    _, T, origin, voxel, g, gv, axes = case
    dims = (24, 20, 12)
    storage = (10, 6, 8)                     # [D0, D1, D2] of a class plane
    G, s = ref.plane_layout(storage, axes)
    if origin is None:      # the map centred on the frame grid's centre, shifted by a third of a voxel
        centre = T @ np.append(np.asarray(g) + np.asarray(G) * gv / 2, 1.0)
        origin = tuple(centre[:3] - np.asarray(dims) * voxel / 2 + voxel / 3)
    off, f = run_emul(emul, T, origin, voxel, dims, g, gv, G, s)
    R = np.linalg.inv(np.asarray(T, np.float64))
    fr, inside = ref.frame_index(R, np.asarray(origin, np.float64), voxel, dims, np.asarray(g, np.float64), gv, G)
    assert np.array_equal(np.moveaxis(fr, 0, -1), f)               # every index, bit for bit
    assert np.array_equal(off >= 0, inside)
    fi = np.moveaxis(fr, 0, -1).astype(np.int64)
    want = fi[..., 0] * s[0] + fi[..., 1] * s[1] + fi[..., 2] * s[2]
    assert np.array_equal(off[inside], want[inside])
    assert 0 < int(inside.sum()) < inside.size or case[0].startswith("identity")


def test_face_centres_take_the_upper_voxel(emul):
    """a centre exactly on a face belongs to the voxel above it (floor), in the kernel and the oracle alike"""
    dims, G, s = (8, 8, 8), (4, 4, 4), (16, 4, 1)
    off, f = run_emul(emul, np.eye(4), (0.0, 0.0, 0.0), 0.5, dims, (0.25, 0.25, 0.25), 0.5, G, s)
    # centre of map voxel i: 0.5 i + 0.25 = the frame face 0.25 + 0.5 i exactly
    assert np.array_equal(f[:, 0, 0, 0], np.arange(8, dtype=np.float64))
    assert (off[:4, :4, :4] >= 0).all() and (off[4:] < 0).all()


@pytest.mark.parametrize("seed", range(6))
def test_box_is_conservative(emul, seed):
    """brute force over small maps the frame grid lies partly outside of: no voxel outside the box is observed"""
    rng = np.random.default_rng(100 + seed)
    dims = tuple(int(v) for v in rng.integers(6, 18, 3))
    voxel = rng.uniform(0.2, 0.5)
    G = tuple(int(v) for v in rng.integers(3, 9, 3))
    gv = rng.uniform(0.2, 0.6)
    s = (G[1] * G[2], G[2], 1)
    for trial in range(8):
        yaw = [0.0, np.pi / 2, np.pi, rng.uniform(-np.pi, np.pi)][trial % 4]
        T = rigid(yaw, rng.uniform(-2, 2 + np.array(dims) * voxel), rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4))
        g = rng.uniform(-1, 1, 3)
        off, _ = run_emul(emul, T, (0.0, 0.0, 0.0), voxel, dims, g, gv, G, s)
        box = fusion.frame_box(T, g, gv, G, np.zeros(3), voxel, dims)
        inb = np.zeros(dims, bool)
        inb[box[0]:box[1], box[2]:box[3], box[4]:box[5]] = True
        assert not (off >= 0)[~inb].any(), (seed, trial, box)
        assert all(0 <= box[2 * a] <= box[2 * a + 1] <= dims[a] for a in range(3))


def test_shift_oracle():
    a = np.arange(2 * 4 * 3 * 5, dtype=np.float32).reshape(2, 4, 3, 5)
    out = ref.shift(a, (1, -1, 2))
    assert out[0, 0, 1, 0] == a[0, 1, 0, 2] and out[1, 2, 2, 2] == a[1, 3, 1, 4]
    assert (out[:, 3] == 0).all() and (out[:, :, 0] == 0).all() and (out[..., 3:] == 0).all()
    assert not ref.shift(a, (4, 0, 0)).any()


# ---- argument refusals of the entry points, without a device ---------------------------------------------------------
def _lib_built():
    _build.build()
    return _lib.lib()


def _integrate_args(**k):
    buf = np.zeros(64, np.float32)
    p = buf.ctypes.data
    a = dict(acc=p, count=p, C=20, MX=4, MY=4, MZ=2, voxel=0.2, origin=np.zeros(3), probs=p,
             strides=np.array([32, 8, 2, 1], np.int64), fov=None, GX=4, GY=4, GZ=2, grid_origin=np.zeros(3),
             grid_voxel=0.2, R=np.eye(4)[:3].copy(), min_prob=1e-3, box=np.array([0, 4, 0, 4, 0, 2], np.int32))
    a.update(k)
    keep = [buf] + [v for v in a.values() if isinstance(v, np.ndarray)]
    ptr = lambda v: v.ctypes.data if isinstance(v, np.ndarray) else v      # noqa: E731
    args = (a["acc"], a["count"], a["C"], a["MX"], a["MY"], a["MZ"], a["voxel"], ptr(a["origin"]), a["probs"],
            ptr(a["strides"]), a["fov"], a["GX"], a["GY"], a["GZ"], ptr(a["grid_origin"]), a["grid_voxel"],
            ptr(a["R"]), a["min_prob"], ptr(a["box"]), None)
    return args, keep


INTEGRATE_BAD = {
    "acc": dict(acc=None), "count": dict(count=None), "probs": dict(probs=None), "origin": dict(origin=None),
    "R_null": dict(R=None), "box_null": dict(box=None), "C0": dict(C=0), "C65": dict(C=65), "MX": dict(MX=0),
    "GZ": dict(GZ=-1), "voxel": dict(voxel=0.0), "voxel_nan": dict(voxel=float("nan")),
    "grid_voxel": dict(grid_voxel=float("inf")), "min_prob0": dict(min_prob=0.0), "min_prob2": dict(min_prob=2.0),
    "min_prob_nan": dict(min_prob=float("nan")), "R_nan": dict(R=np.array([np.nan] + [0.0] * 11)),
    "origin_inf": dict(origin=np.array([0.0, np.inf, 0.0])), "box_hi": dict(box=np.array([0, 5, 0, 4, 0, 2], np.int32)),
    "box_neg": dict(box=np.array([0, 4, -1, 4, 0, 2], np.int32)),
    "box_flip": dict(box=np.array([0, 4, 0, 4, 2, 1], np.int32)),
    "stride": dict(strides=np.array([32, -8, 2, 1], np.int64)),
}


@pytest.mark.parametrize("case", sorted(INTEGRATE_BAD))
def test_integrate_refusals(case):
    L = _lib_built()
    args, keep = _integrate_args(**INTEGRATE_BAD[case])
    assert L.occd_scene_map_integrate(*args) == _lib.ERR_ARG, case
    assert L.occd_last_error().startswith(b"occd_scene_map_integrate: "), L.occd_last_error()


def test_integrate_empty_box_launches_nothing():
    """an empty box answers OK before any CUDA call (host pointers would fault a launch)"""
    L = _lib_built()
    args, keep = _integrate_args(box=np.array([2, 2, 0, 4, 0, 2], np.int32))
    assert L.occd_scene_map_integrate(*args) == 0


def test_shift_and_mark_refusals():
    L = _lib_built()
    a, b = np.zeros(8, np.float32), np.zeros(8, np.float32)
    d = np.zeros(3, np.int32)
    A, B, D = a.ctypes.data, b.ctypes.data, d.ctypes.data
    for args in [(None, A, B, B, 2, 2, 2, 2, D), (A, A, B, B, 0, 2, 2, 2, D), (A, A, B, B, 65, 2, 2, 2, D),
                 (A, A, B, B, 2, 0, 2, 2, D), (A, A, B, B, 2, 2, 2, 2, None), (A, A, A, B, 2, 2, 2, 2, D)]:
        assert L.occd_scene_map_shift(*args, None) == _lib.ERR_ARG, args
        assert L.occd_last_error().startswith(b"occd_scene_map_shift: ")
    for args in [(None, A, 8, 255), (A, None, 8, 255), (A, A, 0, 255), (A, A, 8, -1), (A, A, 8, 65536)]:
        assert L.occd_scene_map_mark_unobserved(*args, None) == _lib.ERR_ARG, args
        assert L.occd_last_error().startswith(b"occd_scene_map_mark_unobserved: ")


# ---- SceneMap and fuse_frames: host-side refusals -----------------------------------------------------------------------
def _cpu_map(C=4, dims=(4, 4, 2)):
    """a SceneMap whose buffers live on the CPU: every refusal of integrate is decided before the library is called"""
    m = object.__new__(fusion.SceneMap)
    m.n_classes, m.dims, m.voxel, m.min_prob = C, dims, 0.2, 1e-3
    m.origin, m.device = np.zeros(3), torch.device("cpu")
    m._acc = torch.zeros((C,) + dims)
    m._count = torch.zeros(dims, dtype=torch.int32)
    m._spare = None
    return m


def test_scene_map_constructor_refusals():
    for kw, msg in [(dict(n_classes=0), "n_classes"), (dict(n_classes=65), "n_classes"),
                    (dict(dims=(4, 0, 2)), "dims"), (dict(dims=(4, 4)), "dims"), (dict(voxel=0.0), "voxel"),
                    (dict(voxel=float("nan")), "voxel"), (dict(origin=(0, 0)), "origin"),
                    (dict(origin=(0, np.inf, 0)), "origin"), (dict(min_prob=0.0), "min_prob"),
                    (dict(min_prob=1.5), "min_prob"), (dict(device="cpu"), "CUDA")]:
        a = dict(n_classes=4, dims=(4, 4, 2), voxel=0.2, origin=(0, 0, 0), device="cuda")
        a.update(kw)
        with pytest.raises(ValueError, match=msg):
            fusion.SceneMap(**a)


def test_integrate_refuses_on_the_host(monkeypatch):
    called = []
    monkeypatch.setattr(_lib, "lib", lambda: called.append(1))
    m = _cpu_map()
    p = torch.zeros(4, 4, 4, 2, dtype=torch.float16)
    with pytest.raises(TypeError, match="float16"):
        m.integrate(p.float(), np.eye(4), (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="probs on"):
        m.integrate(p.to("meta"), np.eye(4), (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="contiguous"):
        m.integrate(p[0], np.eye(4), (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="contiguous"):
        m.integrate(p.transpose(1, 2), np.eye(4), (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="holds 5 classes"):
        m.integrate(torch.zeros(5, 4, 4, 2, dtype=torch.float16), np.eye(4), (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="axes"):
        m.integrate(p, np.eye(4), (0, 0, 0), 0.2, axes="zyx")
    for bad in (np.eye(3), np.full((4, 4), np.nan), np.zeros((4, 4)), torch.eye(4)[:3]):
        with pytest.raises(ValueError, match="pose"):
            m.integrate(p, bad, (0, 0, 0), 0.2)
    with pytest.raises(ValueError, match="grid_origin"):
        m.integrate(p, np.eye(4), (0, 0), 0.2)
    with pytest.raises(ValueError, match="grid_voxel"):
        m.integrate(p, np.eye(4), (0, 0, 0), -0.2)
    with pytest.raises(TypeError, match="fov_mask"):
        m.integrate(p, np.eye(4), (0, 0, 0), 0.2, fov_mask=np.ones(32, bool))
    with pytest.raises(ValueError, match="one class plane|a class plane"):
        m.integrate(p, np.eye(4), (0, 0, 0), 0.2, fov_mask=torch.ones(31, dtype=torch.bool))
    with pytest.raises(ValueError, match="shift"):
        m.shift((1, 0.5, 0))
    with pytest.raises(ValueError, match="unknown"):
        m.classes(unknown=70000)
    assert not called


@pytest.fixture(scope="module")
def kitti_model():
    if os.path.join(ROOT, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
    import shipped_configs
    m, _, _ = shipped_configs.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=(96, 320), full=(64, 64, 16))
    return m


def _kitti(V=2, H=96, W=320):
    return {"img": np.zeros((V, H, W, 3), np.uint8), "cam_k": np.stack([np.eye(3)] * V),
            "T_velo_2_cam": np.stack([np.eye(4)] * V), "img_hw": (H, W)}


def test_fuse_frames_refusals(kitti_model, monkeypatch):
    m = kitti_model
    ran = []
    monkeypatch.setattr(m, "_run_frames", lambda *a, **k: ran.append(1))
    monkeypatch.setattr(m, "_run_frame", lambda *a, **k: ran.append(1))
    smap = _cpu_map(C=m.n_classes)
    with pytest.raises(ValueError, match="1 poses for 2 frames"):
        m.fuse_frames(smap, [_kitti(), _kitti()], [np.eye(4)])
    with pytest.raises(TypeError, match="SceneMap"):
        m.fuse_frames(object(), [_kitti()], [np.eye(4)])
    with pytest.raises(ValueError, match="the map holds 4 classes"):
        m.fuse_frames(_cpu_map(C=4), [_kitti()], [np.eye(4)])
    with pytest.raises(ValueError, match="pose"):
        m.fuse_frames(smap, [_kitti(), _kitti()], [np.eye(4), np.full((4, 4), np.inf)])
    with pytest.raises(ValueError, match="pose"):
        m.fuse_frames(smap, _kitti(), np.eye(3))
    from occdepth_b200.parallel import SimSlabGroup
    m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
    try:
        with pytest.raises(NotImplementedError, match="slab"):
            m.fuse_frames(smap, [_kitti()], [np.eye(4)])
    finally:
        m.__dict__.pop("slab_ctx", None)
    assert not ran
