"""Voxel -> pixel projection (SURVEY 8f row 2): oracle restatement vs the committed reference outputs, and the CUDA
kernel's __host__ __device__ body (csrc/vox2pix.cuh, run on the CPU by tests/host_emul/vox2pix_emul.cu) vs both --
bit for bit, indices AND the float depth."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import projection

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "vox2pix.pt"))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("v2p_emul") / "libv2p_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "vox2pix_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.vox2pix_emulate.restype = C.c_int
    lib.vox2pix_emulate.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double] + [C.c_int] * 5 + \
                                   [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def case_args(c):
    return (c["cam_E"].numpy(), c["cam_k"].numpy(), c["vox_origin"].numpy(), c["voxel_size"], c["img_W"], c["img_H"],
            c["scene_size"], c["pattern_id"])


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_matches_reference_outputs(name):
    c = GOLD[name]
    pix, fov, z = projection.vox2pix(*case_args(c))
    assert pix.dtype == np.int64 and fov.dtype == np.bool_ and z.dtype == c["pix_z"].numpy().dtype
    assert np.array_equal(pix, c["pix"].numpy())
    assert np.array_equal(fov, c["fov"].numpy())
    assert np.array_equal(z, c["pix_z"].numpy(), equal_nan=True)


def run_emul(lib, cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id):
    from occdepth_b200.data import PIXEL_PATTERNS, volume_dims
    X, Y, Z = (int(v) for v in volume_dims(vox_origin, voxel_size, scene_size))
    f32 = np.asarray(cam_E).dtype == np.float32
    E = np.ascontiguousarray(np.asarray(cam_E).astype(np.float32 if f32 else np.float64))
    k32 = np.ascontiguousarray(np.asarray(cam_k).astype(np.float32))
    o32 = np.ascontiguousarray(np.asarray(vox_origin).astype(np.float32))
    pat = np.ascontiguousarray(np.asarray(PIXEL_PATTERNS[pattern_id], dtype=np.int32))
    N, P = X * Y * Z, len(pat)
    pix = np.full((N, P, 2), -7, dtype=np.int64)
    fov = np.full((N, P), 3, dtype=np.uint8)
    z = np.full(N, np.nan, dtype=np.float32 if f32 else np.float64)
    rc = lib.vox2pix_emulate(E.ctypes.data, 1 if f32 else 0, k32.ctypes.data, o32.ctypes.data, float(voxel_size), X, Y, Z,
                             img_W, img_H, pat.ctypes.data, P, pix.ctypes.data, fov.ctypes.data, z.ctypes.data)
    assert rc == 0
    return pix, fov.astype(bool), z


@pytest.mark.parametrize("name", sorted(GOLD))
def test_kernel_body_matches_reference_outputs(emul, name):
    c = GOLD[name]
    pix, fov, z = run_emul(emul, *case_args(c))
    assert np.array_equal(pix, c["pix"].numpy())
    assert np.array_equal(fov, c["fov"].numpy())
    assert np.array_equal(z, c["pix_z"].numpy(), equal_nan=True)      # float depth too: same FMA chain as the BLAS dot


def test_in_plane_centres_take_the_x86_conversion_path():
    """centres exactly in the camera plane divide by zero; the compiled reference's int() then yields INT64_MIN"""
    c = GOLD["plane_p1"]
    z = c["pix_z"].numpy()
    assert (z == 0).any() and (z < 0).any()
    bad = c["pix"].numpy()[z == 0][:, 0, :]
    assert (bad == np.iinfo(np.int64).min).any()
    assert not c["fov"].numpy()[z <= 0].any()


@pytest.mark.parametrize("pattern_id", range(9))
def test_kernel_body_matches_oracle_all_patterns(emul, pattern_id):
    """the full KITTI lift grid geometry (128x128x16 at 0.4 m would be slow in the oracle: use 32x32x8) for every
    pattern of fusion.py:238-330"""
    c = GOLD["kitti_p0"]
    args = list(case_args(c))
    args[6], args[7] = (12.8, 12.8, 3.2), pattern_id
    want = projection.vox2pix(*args)
    got = run_emul(emul, *args)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
