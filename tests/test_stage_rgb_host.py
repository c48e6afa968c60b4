"""The camera-frame staging arithmetic of csrc/normalize_rgb.cuh run on the CPU, bit for bit against the datasets'
host route: `occd_stage_rgb_u8_cl` = numpy normalize_rgb (kitti_dataset.py:376-402) followed by the activation type's
rounding (TF32 round-to-nearest-away, or bf16 round-to-nearest-even) in the channels-last layout with zero pad
channels, for every (value, channel), cropped and strided images; `occd_depth_u16_to_f32` = NYU's load_depth
(nyu_dataset.py:42-48) for all 65 536 uint16 values."""
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
    out = tmp_path_factory.mktemp("stage_emul") / "libstage_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "stage_rgb_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.stage_rgb_emulate.restype = C.c_int
    lib.stage_rgb_emulate.argtypes = [C.c_void_p, C.c_longlong, C.c_longlong] + [C.c_int] * 3 + \
        [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.depth_emulate.restype = C.c_int
    lib.depth_emulate.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_double, C.c_float]
    return lib


def host_normalize(img_u8, H, W):
    """normalize_rgb((np.array(img, np.float32) / 255.0)[:H, :W]) in numpy: ToTensor's HWC -> CHW and Normalize's
    (x - mean) / std, float32 throughout -> (H, W, 3)"""
    img = np.array(img_u8, dtype=np.float32) / 255.0
    img = img[:H, :W, :]
    return (img - np.asarray(MEAN, dtype=np.float32)) / np.asarray(STD, dtype=np.float32)


def to_act(x, dtype):
    """the rounding occd_planar_to_cl applies: TF32 (cvt.rna: ties away from zero) or bf16 (nearest even), as bits"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if dtype == "tf32":
        u = x.view(np.uint32)
        return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32).view(np.uint32)
    return torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def expected(imgs, H, W, dtype, cstride=8):
    out = np.zeros((len(imgs), H, W, cstride), dtype=np.uint32 if dtype == "tf32" else np.uint16)
    for i, im in enumerate(imgs):
        out[i, :, :, :3] = to_act(host_normalize(im, H, W), dtype)
    return out


def run(lib, buf, img_stride, row_stride, n, H, W, dtype, cstride=8):
    """buf: the uint8 bytes the n images live in; returns the staged buffer's bits (n, H, W, cstride)"""
    et = np.uint32 if dtype == "tf32" else np.uint16
    out = np.full((n, H, W, cstride), 0xABCD, dtype=et)          # garbage: the pad channels must be written
    m, s = np.asarray(MEAN, dtype=np.float32), np.asarray(STD, dtype=np.float32)
    buf = np.ascontiguousarray(buf)
    assert lib.stage_rgb_emulate(buf.ctypes.data, img_stride, row_stride, n, H, W, m.ctypes.data, s.ctypes.data,
                                 out.ctypes.data, 0 if dtype == "tf32" else 1, cstride) == 0
    return out


@pytest.mark.parametrize("dtype", ["tf32", "bf16"])
def test_every_value_and_channel(emul, dtype):
    img = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)          # (1, 256, 3)
    got = run(emul, img, img.nbytes, 256 * 3, 1, 1, 256, dtype)
    assert np.array_equal(got, expected([img], 1, 256, dtype))


@pytest.mark.parametrize("dtype", ["tf32", "bf16"])
def test_cropped_strided_images(emul, dtype):
    """two images of raw size 37 x 53, cropped to 30 x 41 (odd W), rows padded to 170 bytes, images 7000 bytes apart;
    a channel stride of 16 gets a second all-zero channel vector"""
    g = np.random.default_rng(0)
    H0, W0, H, W, rs, ist = 37, 53, 30, 41, 170, 7000
    buf = g.integers(0, 256, size=2 * ist, dtype=np.uint8)
    imgs = [np.lib.stride_tricks.as_strided(buf[i * ist:], shape=(H0, W0, 3), strides=(rs, 3, 1)) for i in range(2)]
    for cstride in (8, 16):
        got = run(emul, buf, ist, rs, 2, H, W, dtype, cstride)
        assert np.array_equal(got, expected(imgs, H, W, dtype, cstride)), cstride


def test_host_normalize_is_the_reference_transform():
    """the numpy restatement above equals torchvision's ToTensor + Normalize, the reference's own transform"""
    from torchvision import transforms
    g = np.random.default_rng(1)
    img = g.integers(0, 256, size=(19, 23, 3), dtype=np.uint8)
    t = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=MEAN, std=STD)])
    want = t((np.array(img, dtype=np.float32) / 255.0)[:17, :21]).numpy().transpose(1, 2, 0)
    assert np.array_equal(host_normalize(img, 17, 21), want)


def load_depth(depth, maxDepth=10, divisor=8000.0):
    """nyu_dataset.py:42-48 after skimage.io.imread (divisor 8000)"""
    depth = depth / divisor
    depth = depth.astype("float32")
    depth[depth > maxDepth] = maxDepth
    depth[depth < 0] = 0
    return depth


@pytest.mark.parametrize("divisor", [8000.0, 3000.0])
def test_depth_every_uint16(emul, divisor):
    """NYU's scale (65535 / 8000 < 10: the clamp never fires) and a smaller divisor whose top values clamp"""
    u = np.arange(65536, dtype=np.uint16)
    got = np.full(u.shape, np.nan, dtype=np.float32)
    assert emul.depth_emulate(u.ctypes.data, got.ctypes.data, u.size, divisor, 10.0) == 0
    want = load_depth(u, divisor=divisor)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert got[int(divisor)] == 1.0 and (got.max() == 10.0) == (divisor < 6553.5)
