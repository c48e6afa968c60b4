"""The camera-format staging of csrc/normalize_rgb.cuh (`occd_stage_camera_u8_cl`) run on the CPU, bit for bit
against OpenCV's host route: `normalize_rgb(cv2.remap(cv2.cvtColor(img, ...), mx, my, INTER_LINEAR,
BORDER_CONSTANT 0))` rounded to the activation type, for every (Y, U, V) triple, every remap fraction cell, map
entries at and beyond every edge and non-finite ones, and RGB / BGR / NV12 with and without maps at odd crop sizes.
Also the entry point's argument checks, which run before any device is touched."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from test_stage_rgb_host import MEAN, STD, ROOT, host_normalize, to_act  # noqa: E402

FMT = {"rgb": 0, "bgr": 1, "nv12": 2}


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("camera_emul") / "libcamera_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "stage_camera_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.stage_camera_emulate.restype = C.c_int
    lib.stage_camera_emulate.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong] + \
        [C.c_int] * 5 + [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.remap_table.argtypes = [C.c_void_p]
    return lib


def lut(dtype):
    """the staged bits of every uint8 value in every channel: [3][256]"""
    v = np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, axis=2)
    return to_act(host_normalize(v, 1, 256), dtype).reshape(256, 3).T.copy()


def expected(rgb, dtype, cstride=8):
    """rgb: uint8 (n, H, W, 3) -> the staged buffer's bits (n, H, W, cstride)"""
    t = lut(dtype)
    out = np.zeros(rgb.shape[:3] + (cstride,), dtype=t.dtype)
    for c in range(3):
        out[..., c] = t[c][rgb[..., c]]
    return out


def run(lib, buf, fmt, img_stride, row_stride, n, H0, W0, H, W, dtype, maps=None, uv_offset=0, cstride=8):
    et = np.uint32 if dtype == "tf32" else np.uint16
    out = np.full((n, H, W, cstride), 0xABCD, dtype=et)
    m, s = np.asarray(MEAN, dtype=np.float32), np.asarray(STD, dtype=np.float32)
    buf = np.ascontiguousarray(buf)
    mp = None if maps is None else np.ascontiguousarray(maps, dtype=np.float32)
    assert lib.stage_camera_emulate(buf.ctypes.data, FMT[fmt], img_stride, row_stride, uv_offset, n, H0, W0, H, W,
                                    None if mp is None else mp.ctypes.data, 0 if mp is None else 2 * H * W,
                                    m.ctypes.data, s.ctypes.data, out.ctypes.data, 0 if dtype == "tf32" else 1,
                                    cstride) == 0
    return out


def cv_remap(rgb, mx, my):
    return cv2.remap(rgb, mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def test_every_yuv_triple(emul):
    """all 256^3 (Y, U, V): per U one NV12 image whose 2x2 blocks hold 4 Y values under one (U, V) sample"""
    W0 = 256 * 64 * 2                        # 256 V values x 64 blocks (4 Y each) x 2 columns
    blk = np.arange(W0 // 2)
    V, g = blk // 64, blk % 64
    Y = np.zeros((2, W0), np.uint8)
    for r in range(2):
        for c in range(2):
            Y[r, 2 * blk + c] = 4 * g + 2 * r + c
    want_lut = lut("tf32")
    for U in range(256):
        uv = np.empty((1, W0), np.uint8)
        uv[0, 0::2], uv[0, 1::2] = U, V
        nv12 = np.concatenate([Y, uv])            # OpenCV's NV12 layout (H0 * 3 / 2, W0)
        got = run(emul, nv12, "nv12", nv12.nbytes, W0, 1, 2, W0, 2, W0, "tf32", uv_offset=2 * W0)
        rgb = cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12)
        for c in range(3):
            assert np.array_equal(got[0, :, :, c], want_lut[c][rgb[..., c]]), (U, c)
        assert not got[..., 3:].any()


def test_remap_table_is_opencv_bilinear(emul):
    """every cell's four weights sum to 32768 and are OpenCV's bilinear products of the 1/32 fractions"""
    t = np.zeros((1024, 4), np.uint16)
    emul.remap_table(t.ctypes.data)
    fy, fx = np.divmod(np.arange(1024), 32)
    want = np.stack([(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx], 1) * 32
    assert np.array_equal(t.astype(np.int64), want) and (t.astype(np.int64).sum(1) == 32768).all()


@pytest.mark.parametrize("dtype", ["tf32", "bf16"])
def test_every_fraction_cell(emul, dtype):
    """a 32 x 32 output whose pixel (fy, fx) samples fraction cell (fy, fx) between random interior taps"""
    g = np.random.default_rng(3)
    H0, W0 = 23, 29
    rgb = g.integers(0, 256, size=(H0, W0, 3), dtype=np.uint8)
    fy, fx = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    mx = (g.integers(0, W0 - 1, size=(32, 32)) + fx / 32.0).astype(np.float32)
    my = (g.integers(0, H0 - 1, size=(32, 32)) + fy / 32.0).astype(np.float32)
    got = run(emul, rgb, "rgb", rgb.nbytes, W0 * 3, 1, H0, W0, 32, 32, dtype, maps=np.stack([mx, my]))
    assert np.array_equal(got, expected(cv_remap(rgb, mx, my)[None], dtype))


def test_map_edges(emul):
    """sources from two pixels before to two past every edge in 1/64 steps, partly outside (black taps), and
    entries halfway between two 1/32 cells (rounded half to even)"""
    g = np.random.default_rng(4)
    H0, W0 = 9, 13
    rgb = g.integers(1, 256, size=(H0, W0, 3), dtype=np.uint8)
    xs = np.arange(-2 * 64, (W0 + 2) * 64 + 1) / 64.0
    ys = np.arange(-2 * 64, (H0 + 2) * 64 + 1) / 64.0
    for mx, my in ((xs[None, :], np.full((1, xs.size), 4.5)), (np.full((1, ys.size), 6.25), ys[None, :]),
                   (xs[None, :], np.resize(ys, xs.size)[None, :])):
        mx, my = mx.astype(np.float32), my.astype(np.float32)
        H, W = mx.shape
        got = run(emul, rgb, "rgb", rgb.nbytes, W0 * 3, 1, H0, W0, H, W, "tf32", maps=np.stack([mx, my]))
        want = cv_remap(rgb, mx, my)
        assert np.array_equal(got, expected(want[None], "tf32"))
    assert not want[0, :10].any()                 # fully outside: black


def test_non_finite_and_huge_map_entries(emul):
    """NaN, +-inf and +-1e30 in either coordinate: OpenCV gives black, and so does the staging"""
    H0, W0 = 6, 8
    rgb = np.full((H0, W0, 3), 200, np.uint8)
    bad = np.array([np.nan, np.inf, -np.inf, 1e30, -1e30, 3e9, -3e9, 7e7], np.float32)
    ok = np.float32(2.5)
    mx = np.concatenate([bad, np.full(bad.size, ok)])[None, :].astype(np.float32)
    my = np.concatenate([np.full(bad.size, ok), bad])[None, :].astype(np.float32)
    got = run(emul, rgb, "rgb", rgb.nbytes, W0 * 3, 1, H0, W0, 1, mx.shape[1], "tf32", maps=np.stack([mx, my]))
    want = cv_remap(rgb, mx, my)
    assert not want.any()                         # pinned: OpenCV writes black for every such entry
    assert np.array_equal(got, expected(want[None], "tf32"))


def _nv12_frames(g, n, H0, W0, pad_rows, row_stride, img_stride):
    """n NV12 images in one buffer: luma rows padded to row_stride, luma height padded by pad_rows (as decoder
    surfaces are), images img_stride apart -> (buffer, uv_offset, [OpenCV's (H0 * 3 / 2, W0) array per image])"""
    uv_offset = (H0 + pad_rows) * row_stride
    buf = g.integers(0, 256, size=n * img_stride, dtype=np.uint8)
    arrays = []
    for i in range(n):
        base = buf[i * img_stride:]
        luma = np.lib.stride_tricks.as_strided(base, shape=(H0, W0), strides=(row_stride, 1))
        chroma = np.lib.stride_tricks.as_strided(base[uv_offset:], shape=(H0 // 2, W0), strides=(row_stride, 1))
        arrays.append(np.concatenate([luma, chroma]))
    return buf, uv_offset, arrays


@pytest.mark.parametrize("dtype", ["tf32", "bf16"])
@pytest.mark.parametrize("fmt", ["rgb", "bgr", "nv12"])
@pytest.mark.parametrize("maps", [False, True])
def test_formats_cropped_strided(emul, dtype, fmt, maps):
    """two raw 38 x 54 images in padded rows, cropped (or remapped) to an odd 29 x 41; the maps hold a lens
    distortion from cv2.initUndistortRectifyMap, with some sources outside the image"""
    g = np.random.default_rng(5)
    n, H0, W0, H, W = 2, 38, 54, 29, 41
    if fmt == "nv12":
        rs = 64
        buf, uv_off, arrays = _nv12_frames(g, n, H0, W0, 2, rs, 4000)
        rgbs = [cv2.cvtColor(a, cv2.COLOR_YUV2RGB_NV12) for a in arrays]
        ist = 4000
    else:
        rs, ist, uv_off = 170, 7000, 0
        buf = g.integers(0, 256, size=n * ist, dtype=np.uint8)
        raw = [np.lib.stride_tricks.as_strided(buf[i * ist:], shape=(H0, W0, 3), strides=(rs, 3, 1))
               for i in range(n)]
        rgbs = [np.ascontiguousarray(r[..., ::-1] if fmt == "bgr" else r) for r in raw]
    if maps:
        mp = []
        for i in range(n):
            K = np.array([[40.0, 0, 27 + i], [0, 40.0, 19], [0, 0, 1]])
            mx, my = cv2.initUndistortRectifyMap(K, np.array([-0.3, 0.1, 0.001, -0.002, 0.0]), None, K, (W, H),
                                                 cv2.CV_32FC1)
            mp.append(np.stack([mx - 3.3, my + 0.7]))
        mp = np.stack(mp).astype(np.float32)
        want = np.stack([cv_remap(r, m[0], m[1]) for r, m in zip(rgbs, mp)])
    else:
        mp = None
        want = np.stack([r[:H, :W] for r in rgbs])
    for cstride in (8, 16):
        got = run(emul, buf, fmt, ist, rs, n, H0, W0, H, W, dtype, maps=mp, uv_offset=uv_off, cstride=cstride)
        assert np.array_equal(got, expected(want, dtype, cstride)), cstride


def test_rgb_without_maps_is_the_rgb_staging(emul):
    """format RGB without maps is the datasets' route: the existing staging body's output exactly"""
    from test_stage_rgb_host import expected as rgb_expected
    g = np.random.default_rng(6)
    img = g.integers(0, 256, size=(17, 25, 3), dtype=np.uint8)
    for dtype in ("tf32", "bf16"):
        got = run(emul, img, "rgb", img.nbytes, 75, 1, 17, 25, 15, 23, dtype)
        assert np.array_equal(got, rgb_expected([img], 15, 23, dtype))


# ---- the entry point's argument checks (the library, no device needed: every refusal precedes the launch) --------

def _lib():
    from occdepth_b200 import _build, _lib as L
    _build.build()
    return L.lib()


def _stage(L, fmt=2, img_stride=0, row_stride=64, uv_offset=64 * 38, n=1, H0=38, W0=54, H=29, W=41, maps=None,
           map_stride=0, out=4096, dtype=0, cstride=8):
    m = (C.c_float * 3)(*MEAN)
    s = (C.c_float * 3)(*STD)
    rc = L.occd_stage_camera_u8_cl(4096, fmt, img_stride, row_stride, uv_offset, n, H0, W0, H, W, maps, map_stride,
                                   m, s, out, dtype, cstride, None)
    return rc, (L.occd_last_error() or b"").decode()


@pytest.mark.parametrize("kw, what", [
    (dict(fmt=3), "format"),
    (dict(fmt=-1), "format"),
    (dict(H0=37), "even"),
    (dict(W0=53), "even"),
    (dict(uv_offset=64 * 37), "chroma plane overlaps"),
    (dict(uv_offset=64 * 37 + 53), "chroma plane overlaps"),
    (dict(row_stride=53), "chroma plane overlaps"),
    (dict(n=2, img_stride=64 * 38 + 64 * 18 + 53), "chroma plane overlaps"),
    (dict(maps=4098), "4-byte aligned"),
    (dict(maps=4096, n=2, img_stride=10 ** 6, map_stride=2 * 29 * 41 - 1), "map_stride"),
    (dict(maps=4096, W0=32768, row_stride=32768, uv_offset=32768 * 38), "32767"),
    (dict(H=39), "crop"),
    (dict(fmt=1, row_stride=161), "strides overlap"),
    (dict(fmt=0, n=2, row_stride=162, img_stride=162 * 37 + 161), "strides overlap"),
    (dict(cstride=12), "cstride"),
    (dict(out=4100), "16-byte aligned"),
    (dict(dtype=7), "dtype"),
])
def test_argument_checks(kw, what):
    L = _lib()
    rc, msg = _stage(L, **kw)
    assert rc == 1 and what in msg and msg.startswith("occd_stage_camera_u8_cl"), (kw, rc, msg)


def test_null_arguments_and_the_rgb_entry_point_keeps_its_messages():
    L = _lib()
    m = (C.c_float * 3)(*MEAN)
    assert L.occd_stage_camera_u8_cl(None, 0, 0, 162, 0, 1, 2, 2, 2, 2, None, 0, m, m, 4096, 0, 8, None) == 1
    assert b"null argument" in L.occd_last_error()
    assert L.occd_stage_rgb_u8_cl(4096, 0, 162, 1, 2, 2, 3, 2, m, m, 4096, 0, 8, None) == 1
    assert L.occd_last_error() == b"occd_stage_rgb_u8_cl: the crop must lie inside the image"
    assert L.occd_stage_rgb_u8_cl(4096, 0, 5, 1, 2, 2, 2, 2, m, m, 4096, 0, 8, None) == 1
    assert L.occd_last_error() == b"occd_stage_rgb_u8_cl: strides overlap the rows / images"
