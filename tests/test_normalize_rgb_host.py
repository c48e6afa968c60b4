"""Image pre-processing of the datasets (kitti_dataset.py:164-171,376-402) vs the kernel body of
csrc/normalize_rgb.cuh run on the CPU: every one of the 256 x 3 possible (value, channel) results, and a cropped
image, bit for bit against torchvision's ToTensor + Normalize applied the way the reference applies it."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("nrm_emul") / "libnrm_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "normalize_rgb_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.normalize_rgb_emulate.restype = C.c_int
    lib.normalize_rgb_emulate.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_void_p]
    return lib


def reference_transform(img_u8, H, W):
    """exactly the reference's sequence (kitti_dataset.py:376-378,402) with torchvision's own transforms"""
    from torchvision import transforms
    normalize_rgb = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=MEAN, std=STD)])
    img = np.array(img_u8, dtype=np.float32) / 255.0
    img = img[:H, :W, :]
    return normalize_rgb(img)


def run(lib, img_u8, H, W):
    H0, W0 = img_u8.shape[:2]
    out = np.full((3, H, W), np.nan, dtype=np.float32)
    m, s = np.asarray(MEAN, dtype=np.float32), np.asarray(STD, dtype=np.float32)
    src = np.ascontiguousarray(img_u8)
    assert lib.normalize_rgb_emulate(src.ctypes.data, out.ctypes.data, H0, W0, H, W, m.ctypes.data, s.ctypes.data) == 0
    return out


def test_every_value_and_channel(emul):
    img = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)          # (1, 256, 3)
    assert np.array_equal(run(emul, img, 1, 256), reference_transform(img, 1, 256).numpy())


def test_cropped_image(emul):
    g = np.random.default_rng(0)
    img = g.integers(0, 256, size=(37, 53, 3), dtype=np.uint8)
    got = run(emul, img, 30, 41)
    want = reference_transform(img, 30, 41).numpy()
    assert got.dtype == want.dtype == np.float32 and got.shape == want.shape
    assert np.array_equal(got, want)
