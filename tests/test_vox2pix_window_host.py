"""Windowed voxel -> pixel projection (occd_vox2pix_range_fwd): the kernel body run over a window of the X-major voxel
order (tests/host_emul/vox2pix_window_emul.cu) is that slice of the whole-grid body (tests/host_emul/vox2pix_emul.cu),
bit for bit, for KITTI and NYU geometry, float32 and float64 poses, one- and many-pixel patterns; and the entry point
refuses windows outside the grid before it touches a device."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "vox2pix.pt"))
_ARGS = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double] + [C.c_int] * 5 + [C.c_void_p, C.c_int] + \
        [C.c_void_p] * 3


def _compile(tmp, src, sym, extra):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp / ("lib%s.so" % sym)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = getattr(C.CDLL(str(out)), sym)
    fn.restype = C.c_int
    fn.argtypes = _ARGS + extra
    return fn


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("v2p_window_emul")
    return (_compile(tmp, "vox2pix_emul.cu", "vox2pix_emulate", []),
            _compile(tmp, "vox2pix_window_emul.cu", "vox2pix_window_emulate", [C.c_longlong, C.c_longlong]))


def _inputs(c, f32, pattern_id):
    from occdepth_b200.data import PIXEL_PATTERNS, volume_dims
    X, Y, Z = (int(v) for v in volume_dims(c["vox_origin"].numpy(), c["voxel_size"], c["scene_size"]))
    E = np.ascontiguousarray(c["cam_E"].numpy().astype(np.float32 if f32 else np.float64))
    k32 = np.ascontiguousarray(c["cam_k"].numpy().astype(np.float32))
    o32 = np.ascontiguousarray(c["vox_origin"].numpy().astype(np.float32))
    pat = np.ascontiguousarray(np.asarray(PIXEL_PATTERNS[pattern_id], dtype=np.int32))
    return (X, Y, Z), E, k32, o32, pat


def _run(fn, c, f32, dims, E, k32, o32, pat, n, *window):
    P = len(pat)
    pix = np.full((n, P, 2), -7, dtype=np.int64)
    fov = np.full((n, P), 3, dtype=np.uint8)
    z = np.full(n, np.nan, dtype=np.float32 if f32 else np.float64)
    rc = fn(E.ctypes.data, 1 if f32 else 0, k32.ctypes.data, o32.ctypes.data, float(c["voxel_size"]), *dims,
            int(c["img_W"]), int(c["img_H"]), pat.ctypes.data, P, pix.ctypes.data, fov.ctypes.data, z.ctypes.data,
            *window)
    assert rc == 0
    return pix, fov, z


def _windows(dims):
    X, Y, Z = dims
    plane, N = Y * Z, X * Y * Z
    return [(0, N), (0, 2 * plane), (0, N // 3), ((X // 2) * plane, 3 * plane), (N // 3, N // 3 + 7),
            (N - 2 * plane, 2 * plane), (N - N // 4, N // 4),
            (0, plane), ((X // 2) * plane, plane), (N - plane, plane),           # one-plane windows
            (N - 1, 1), (5, 1)]


@pytest.mark.parametrize("f32", [False, True], ids=["f64_pose", "f32_pose"])
@pytest.mark.parametrize("name,pattern_id", [("kitti_p0", 0), ("kitti_p3", 3), ("nyu_p8", 0), ("nyu_p8", 8),
                                             ("plane_p1", 1)])
def test_window_is_the_slice_of_the_whole_grid(emul, name, pattern_id, f32):
    whole_fn, window_fn = emul
    c = GOLD[name]
    dims, E, k32, o32, pat = _inputs(c, f32, pattern_id)
    whole = _run(whole_fn, c, f32, dims, E, k32, o32, pat, int(np.prod(dims)))
    for v0, n in _windows(dims):
        got = _run(window_fn, c, f32, dims, E, k32, o32, pat, n, v0, n)
        for g, w in zip(got, whole):
            assert np.array_equal(g, w[v0:v0 + n], equal_nan=True), (name, v0, n)


# ---- the entry point's argument checks (they run before any launch, so no device is needed) ------------------------
def _lib_built():
    from occdepth_b200 import _build, _lib
    _build.build()
    return _lib.lib()


@pytest.mark.parametrize("dims,v0,n", [
    ((4, 3, 2), -1, 1),                # starts before the grid
    ((4, 3, 2), 0, 0),                 # empty
    ((4, 3, 2), 0, -5),
    ((4, 3, 2), 20, 5),                # ends past the grid
    ((4, 3, 2), 24, 1),
    ((4, 3, 2), 1, 1 << 62),           # v0 + n would overflow
    ((0, 3, 2), 0, 1),                 # bad dims
    ((1 << 14, 1 << 14, 1 << 14), 0, 1 << 42),     # more blocks than one grid launch takes
])
def test_range_entry_point_refuses(dims, v0, n):
    from occdepth_b200 import _lib
    L = _lib_built()
    E, k = np.eye(4), np.eye(3, dtype=np.float32)
    o = np.zeros(3, np.float32)
    pat = np.zeros(2, np.int32)
    pix, fov = np.zeros(8, np.int64), np.zeros(8, np.uint8)
    rc = L.occd_vox2pix_range_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, 0.2, *dims, 64, 48, pat.ctypes.data,
                                  1, pix.ctypes.data, fov.ctypes.data, None, v0, n, None)
    assert rc == _lib.ERR_ARG
    assert L.occd_last_error().decode().startswith("occd_vox2pix_range_fwd: ")


def test_whole_grid_entry_point_keeps_its_checks():
    from occdepth_b200 import _lib
    L = _lib_built()
    E, k = np.eye(4), np.eye(3, dtype=np.float32)
    o = np.zeros(3, np.float32)
    pat = np.zeros(2, np.int32)
    pix, fov = np.zeros(8, np.int64), np.zeros(8, np.uint8)
    for dims, P, text in (((0, 3, 2), 1, "dims"), ((4, 3, 2), 26, "pattern size"),
                          ((1 << 14, 1 << 14, 1 << 14), 1, "too many voxels")):
        rc = L.occd_vox2pix_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, 0.2, *dims, 64, 48, pat.ctypes.data,
                                P, pix.ctypes.data, fov.ctypes.data, None, None)
        msg = L.occd_last_error().decode()
        assert rc == _lib.ERR_ARG and msg.startswith("occd_vox2pix_fwd: ") and text in msg, msg


def test_vox2pix_into_checks_the_window():
    """the Python wrapper refuses a window outside the grid and buffers that do not hold it, before any launch"""
    from occdepth_b200 import data as D
    c = GOLD["kitti_p0"]
    args = (c["cam_E"].numpy(), c["cam_k"].numpy(), c["vox_origin"].numpy(), c["voxel_size"], c["img_W"], c["img_H"],
            c["scene_size"], 0)
    N = c["pix"].shape[0]
    pix, fov, z = torch.zeros(16, 1, 2, dtype=torch.int64), torch.zeros(16, 1, dtype=torch.bool), torch.zeros(16)
    with pytest.raises(ValueError, match="voxel_range"):
        D.vox2pix_into(pix, fov, z.double(), *args, voxel_range=(N - 8, 16))
    with pytest.raises(ValueError, match="index grid"):
        D.vox2pix_into(pix, fov, z.double(), *args, voxel_range=(0, 8))
