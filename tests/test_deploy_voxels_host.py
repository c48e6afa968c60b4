"""CPU checks of the occupied-voxel list of model files and of batched camera frames: occd_model_list_voxels refuses
bad arguments before it reads the model or touches a device; the voxel -> pixel body with no pixel output writes the
same FOV mask bytes as with it (tests/host_emul/vox2pix_window_emul.cu); predict_voxels of a list of frames and
LoadedModel.list_voxels refuse bad requests on the host, before any device work."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200.voxels import VoxelList

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib_built():
    _build.build()
    return _lib.lib()


# ---- occd_model_list_voxels: the argument refusals ---------------------------------------------------------------------
def _out(**k):
    buf = np.zeros(16, np.int64)                 # any non-null address: the refusals come before it is read
    p = buf.ctypes.data
    vo = _lib.VoxelOut(capacity=4, voxel_size=0.0, origin=None, count=p, hist=p, index=p, cls=p, xyz=None)
    for name, v in k.items():
        setattr(vo, name, v)
    return vo, buf


@pytest.mark.parametrize("case", ["model", "out", "count", "hist", "index", "cls", "capacity", "voxel_size"])
def test_list_voxels_refuses_before_reading_the_model(case):
    L = _lib_built()
    # a stand-in handle: every refusal below is decided from the arguments alone, before the model is read
    fake = np.zeros(64, np.uint8)
    m = None if case == "model" else fake.ctypes.data
    if case in ("count", "hist", "index", "cls"):
        vo, keep = _out(**{case: None})
    elif case == "capacity":
        vo, keep = _out(capacity=-1)
    elif case == "voxel_size":
        vo, keep = _out(voxel_size=-0.2)
    else:
        vo, keep = _out()
    rc = L.occd_model_list_voxels(m, 1, None if case == "out" else C.byref(vo), None)
    msg = L.occd_last_error().decode()
    assert rc == _lib.ERR_ARG, (case, rc, msg)
    assert msg.startswith("occd_model_list_voxels: "), msg


# ---- the voxel -> pixel body without the pixel output ------------------------------------------------------------------
_ARGS = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double] + [C.c_int] * 5 + [C.c_void_p, C.c_int] + \
        [C.c_void_p] * 3 + [C.c_longlong, C.c_longlong]


@pytest.fixture(scope="module")
def window_emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("v2p_null_pix") / "libv2p_window.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "vox2pix_window_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).vox2pix_window_emulate
    fn.restype = C.c_int
    fn.argtypes = _ARGS
    return fn


def _random_kitti_calib(rng):
    """a KITTI-like camera: a rotation mostly looking along +x of the velodyne frame, a small offset, KITTI-sized
    intrinsics"""
    a, b, c = rng.uniform(-0.08, 0.08, 3)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(c), -np.sin(c)], [0, np.sin(c), np.cos(c)]])
    base = np.array([[0.0, -1, 0], [0, 0, -1], [1, 0, 0]])               # velodyne -> camera axes
    T = np.eye(4)
    T[:3, :3] = base @ Rz @ Ry @ Rx
    T[:3, 3] = rng.uniform(-0.5, 0.5, 3)
    K = np.array([[rng.uniform(600, 800), 0, rng.uniform(580, 640)], [0, rng.uniform(600, 800), rng.uniform(160, 200)],
                  [0, 0, 1]])
    return T, K


@pytest.mark.parametrize("f32", [False, True], ids=["f64_pose", "f32_pose"])
def test_null_pix_writes_the_same_mask(window_emul, f32):
    from occdepth_b200.data import volume_dims
    rng = np.random.default_rng(11 + int(f32))
    origin, scene, voxel = np.array([0.0, -25.6, -2.0]), (51.2, 51.2, 6.4), 0.8
    X, Y, Z = (int(v) for v in volume_dims(origin, voxel, scene))
    N, plane = X * Y * Z, Y * Z
    o32 = np.ascontiguousarray(origin.astype(np.float32))
    pat = np.zeros(2, np.int32)
    for trial in range(4):
        T, K = _random_kitti_calib(rng)
        E = np.ascontiguousarray(T.astype(np.float32 if f32 else np.float64))
        k32 = np.ascontiguousarray(K.astype(np.float32))
        for v0, n in ((0, N), (0, 3 * plane), ((X // 2) * plane, 5 * plane), (N - plane, plane), (N // 3, 77)):
            pix = np.full((n, 1, 2), -7, np.int64)
            fov = np.full(n, 3, np.uint8)
            z = np.full(n, np.nan, np.float32 if f32 else np.float64)
            args = (E.ctypes.data, int(f32), k32.ctypes.data, o32.ctypes.data, voxel, X, Y, Z, 1220, 370,
                    pat.ctypes.data, 1)
            assert window_emul(*args, pix.ctypes.data, fov.ctypes.data, z.ctypes.data, v0, n) == 0
            fov_only = np.full(n, 5, np.uint8)
            z_only = np.full(n, np.nan, z.dtype)
            assert window_emul(*args, None, fov_only.ctypes.data, z_only.ctypes.data, v0, n) == 0
            assert fov_only.tobytes() == fov.tobytes(), (trial, v0, n)
            assert z_only.tobytes() == z.tobytes(), (trial, v0, n)
            mask_alone = np.full(n, 5, np.uint8)
            assert window_emul(*args, None, mask_alone.ctypes.data, None, v0, n) == 0
            assert mask_alone.tobytes() == fov.tobytes(), (trial, v0, n)
            assert 0 < int(fov.sum()) < n or n < plane * 4, (trial, v0, n)     # a real split, not a constant mask


def test_entry_points_take_a_null_pix_but_not_a_null_fov():
    L = _lib_built()
    E, k = np.eye(4), np.eye(3, dtype=np.float32)
    o = np.zeros(3, np.float32)
    pat = np.zeros(2, np.int32)
    rc = L.occd_vox2pix_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, 0.2, 4, 3, 2, 64, 48, pat.ctypes.data, 1,
                            None, None, None, None)
    assert rc == _lib.ERR_ARG and b"null argument" in L.occd_last_error()
    rc = L.occd_vox2pix_range_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, 0.2, 4, 3, 2, 64, 48,
                                  pat.ctypes.data, 1, None, None, None, 0, 24, None)
    assert rc == _lib.ERR_ARG and b"null argument" in L.occd_last_error()
    # with pix NULL the checks after the null check still answer (the window), so pix is not what is refused
    fov = np.zeros(8, np.uint8)
    rc = L.occd_vox2pix_range_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, 0.2, 4, 3, 2, 64, 48,
                                  pat.ctypes.data, 1, None, fov.ctypes.data, None, 20, 5, None)
    assert rc == _lib.ERR_ARG and b"window" in L.occd_last_error()


# ---- predict_voxels of a list of frames: host-side refusals -----------------------------------------------------------
def _kitti(V=2, H=96, W=320, **extra):
    f = {"img": np.zeros((V, H, W, 3), np.uint8), "cam_k": np.stack([np.eye(3)] * V),
         "T_velo_2_cam": np.stack([np.eye(4)] * V), "img_hw": (H, W)}
    f.update(extra)
    return f


@pytest.fixture(scope="module")
def kitti_model():
    if os.path.join(ROOT, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
    import shipped_configs
    m, _, _ = shipped_configs.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=(96, 320), full=(64, 64, 16))
    return m


def test_predict_voxels_list_refusals(kitti_model, monkeypatch):
    m = kitti_model
    ran = []
    monkeypatch.setattr(m, "_run_frames", lambda *a, **k: ran.append(1))
    for bad in (42, "frames", torch.zeros(3)):
        with pytest.raises(TypeError, match="OccDepth.predict_voxels"):
            m.predict_voxels(bad)
    with pytest.raises(TypeError, match="item 1 of the list"):
        m.predict_voxels([_kitti(), 7])
    with pytest.raises(ValueError, match="0 frames"):
        m.predict_voxels([])
    with pytest.raises(ValueError, match="frame 1's V"):
        m.predict_voxels([_kitti(), _kitti(V=1)])
    with pytest.raises(ValueError, match="frame 1's img_hw"):
        m.predict_voxels([_kitti(), _kitti(img_hw=(96, 288))])
    with pytest.raises(ValueError, match="slab_output"):
        m.predict_voxels([_kitti()], slab_output="root")
    from occdepth_b200.parallel import SimSlabGroup
    m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
    try:
        with pytest.raises(NotImplementedError, match="one frame per forward"):
            m.predict_voxels([_kitti(), _kitti()])
        with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
            m.predict_voxels([_kitti()])
    finally:
        m.__dict__.pop("slab_ctx", None)
    assert not ran


# ---- LoadedModel.list_voxels: host-side refusals ----------------------------------------------------------------------
def _unloaded(X=8, Y=8, Z=4, last_n=2):
    """a LoadedModel that holds no file: list_voxels' argument checks run before the library is called"""
    lm = object.__new__(deploy.LoadedModel)
    lm.handle, lm.comm = None, None
    lm.geom = _lib.ModelGeom(X=X, Y=Y, Z=Z)
    lm._last_n = last_n
    return lm


def test_loaded_model_list_voxels_refusals():
    lm = _unloaded()
    N = 8 * 8 * 4
    with pytest.raises(ValueError, match="vox_origin without coordinates"):
        lm.list_voxels(xyz=False, vox_origin=[0, -25.6, -2])
    with pytest.raises(ValueError, match="3 values"):
        lm.list_voxels(vox_origin=[0, 1])
    with pytest.raises(ValueError, match="capacity must be >= 0"):
        lm.list_voxels(capacity=-1)
    out = VoxelList(2, N, 100, True, "cpu")
    with pytest.raises(ValueError, match="another n, capacity or xyz"):
        lm.list_voxels(capacity=50, out=out)
    with pytest.raises(ValueError, match="another n, capacity or xyz"):
        lm.list_voxels(out=out)                             # the default capacity is N
    with pytest.raises(ValueError, match="another n, capacity or xyz"):
        lm.list_voxels(capacity=100, out=out, xyz=False)
    with pytest.raises(ValueError, match="another n, capacity or xyz"):
        lm.list_voxels(n=1, capacity=100, out=out)
