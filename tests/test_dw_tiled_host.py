"""CPU check of the shared-memory-tiled depthwise kernel (csrc/dwconv_tiled.cuh): the kernel's phase functions
are __host__ __device__, so the same tile / halo / stride / ragged-edge index arithmetic that runs on the GPU is
executed here thread by thread (tests/host_emul/dw_tiled_emul.cu) and compared with torch's depthwise conv
(geffnet conv_dw + bn + SiLU + the SE squeeze, unet2d.py:188-196)."""
import ctypes as C
import math
import os
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("dw_emul") / "libdw_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "dw_tiled_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    lib = C.CDLL(str(out))
    lib.dw_tiled_emulate.restype = C.c_int
    lib.dw_tiled_emulate.argtypes = [C.c_void_p] * 5 + [C.c_int] * 15 + [C.POINTER(C.c_int)] * 2
    return lib


def same_pad(n, k, s):
    return max((math.ceil(n / s) - 1) * s + k - n, 0)


CASES = [
    # B, C,  H,  W, K, S, cs_extra, th
    (1, 64, 9, 21, 3, 1, 0, 0),
    (2, 64, 19, 37, 5, 1, 0, 8),
    (1, 64, 19, 37, 5, 1, 0, 16),
    (1, 72, 11, 18, 3, 1, 8, 0),     # ragged channel tile (72 = 64 + 8), padded channel stride
    (1, 32, 23, 33, 3, 1, 0, 0),     # narrow layer -> CVB = 4 shape
    (1, 24, 17, 20, 5, 2, 0, 0),     # narrow + stride 2
    (2, 64, 20, 35, 3, 2, 0, 0),     # stride 2, even / odd extents (TF-SAME pads asymmetrically)
    (1, 128, 21, 34, 5, 2, 0, 0),
    (1, 64, 3, 5, 5, 1, 0, 0),       # image smaller than the filter
]


def round_tf32(t):
    return ((t.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("B,Cn,H,W,K,S,cs_extra,th", CASES)
def test_tiled_dw_matches_torch(emul, B, Cn, H, W, K, S, cs_extra, th, dtype):
    g = torch.Generator().manual_seed(1000 * K + 10 * S + Cn + H)
    cs_in, cs_out = Cn + cs_extra, Cn + cs_extra
    bf16 = dtype == torch.bfloat16
    x = torch.randn(B, H, W, cs_in, generator=g)
    x = x.to(torch.bfloat16) if bf16 else round_tf32(x)
    w = torch.randn(Cn, K, K, generator=g) * 0.3
    bias = torch.randn(Cn, generator=g) * 0.2
    OH, OW = math.ceil(H / S), math.ceil(W / S)
    ph, pw = same_pad(H, K, S), same_pad(W, K, S)
    pt, pl = ph // 2, pw // 2
    wt = w.reshape(Cn, K * K).t().contiguous()                       # [K*K][C], the layout the kernel reads
    out = torch.full((B, OH, OW, cs_out), float("nan")).to(dtype)
    pool = torch.zeros(B, Cn, dtype=torch.int64)
    cvb, tho = C.c_int(), C.c_int()
    rc = emul.dw_tiled_emulate(x.data_ptr(), wt.data_ptr(), bias.data_ptr(), out.data_ptr(), pool.data_ptr(),
                               2 if bf16 else 4, B, H, W, OH, OW, Cn, cs_in, cs_out, K, S, pt, pl, 3, th,
                               C.byref(cvb), C.byref(tho))
    assert rc == 0
    assert cvb.value == (4 if (Cn < 64 or not bf16) else 8)
    if th and cvb.value == 8 and S == 1:
        assert tho.value == th
    xin = x[..., :Cn].float().permute(0, 3, 1, 2)
    xin = F.pad(xin, (pl, pw - pl, pt, ph - pt))
    ref = F.silu(F.conv2d(xin, w[:, None], bias, stride=S, groups=Cn)).permute(0, 2, 3, 1)
    got = out[..., :Cn].float()
    assert torch.isfinite(got).all()
    tol = 1e-2 if bf16 else 1e-3        # one bf16 / TF32 store rounding
    assert torch.allclose(got, ref, rtol=tol, atol=tol), (got - ref).abs().max()
    if not bf16:                        # every stored value is TF32-representable
        assert torch.equal(got, round_tf32(got))
    # the squeeze sums the rounded outputs in 2^-24 fixed point
    want = got.double().sum(dim=(1, 2))
    assert torch.allclose(pool.double() / 2 ** 24, want, rtol=1e-5, atol=1e-3)
    if cs_extra:                                                     # padding lanes of the output are untouched
        assert torch.isnan(out[..., Cn:].float()).all()
