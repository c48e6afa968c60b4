"""Class-map confidence (OCCD_OUT1_CLASS_U16_CONF) on the host.

- The running arg-max and softmax of the class-map epilogues (ClassArg, csrc/conv_common.cuh), compiled for the CPU
  (tests/host_emul/class_conf_emul.cu) and driven in each epilogue's merge order, on random vectors of 2 to 64
  channels with ties, NaN, +-inf and magnitudes near 1e30: the class follows occd_argmax_classes' rule, and the
  confidence is float16(p) or one of its float16 neighbours, p the float64 softmax maximum, NaN exactly where p is.
- Plan creation without a GPU: mode 4 is accepted and refused exactly where mode 3 is, occd_argmax_classes_conf checks
  its arguments, and the engine falls back to logits + occd_argmax_classes_conf.
- The model loader: flag bit 2 needs a class-map role twice the map's length; unknown flag bits are refused."""
import contextlib
import ctypes as C
import io
import os
import shutil
import subprocess
import struct

import numpy as np
import pytest
import torch
import torch.nn as nn

from occdepth_b200 import _build, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 0x100000        # an aligned device address: plan creation never dereferences it


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("class_conf_emul") / "libclass_conf_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "class_conf_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).class_conf_emulate
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return fn


def _emulate(fn, x, order, conf=True):
    x = np.ascontiguousarray(x, np.float32)
    n, Cn = x.shape
    cls = np.zeros(n, np.uint16)
    bits = np.zeros(n, np.uint16)
    assert fn(x.ctypes.data, n, Cn, order, 1 if conf else 0, cls.ctypes.data, bits.ctypes.data) == 0
    return cls, bits.view(np.float16)


def ref_class(x):
    """occd_argmax_classes' rule: the first index of the largest value; NaN in channel 0 wins, later NaNs are skipped"""
    out = np.zeros(len(x), np.int64)
    for i, v in enumerate(x):
        if np.isnan(v[0]):
            continue
        w = np.where(np.isnan(v), -np.inf, v.astype(np.float64))
        out[i] = int(np.argmax(w))
    return out


def check_conf(conf, logits):
    """conf (float16 [n]) against the float64 softmax maximum of logits ([n, C]): float16(p) or a float16 neighbour
    of it, NaN exactly where p is NaN"""
    p = torch.softmax(torch.as_tensor(np.asarray(logits, np.float64)), dim=1).max(dim=1).values.numpy()
    conf = np.asarray(conf, np.float16)
    nan_p = np.isnan(p)
    assert np.array_equal(np.isnan(conf), nan_p), np.flatnonzero(np.isnan(conf) != nan_p)[:10]
    h = p[~nan_p].astype(np.float16)
    c = conf[~nan_p]
    ok = (c == h) | (c == np.nextafter(h, np.float16(np.inf))) | (c == np.nextafter(h, np.float16(-np.inf)))
    assert ok.all(), list(zip(c[~ok][:5], p[~nan_p][~ok][:5]))


def _vectors(Cn, rng, n=400):
    x = rng.normal(0, 3, (n, Cn)).astype(np.float32)
    x[:40] = np.round(x[:40])                                  # ties
    x[40:60] = x[40:60] * 1e-4                                  # near-uniform: p close to 1 / C
    x[60:80] *= 1e29                                            # magnitudes of about 1e30
    x[80:90, 0] = np.nan                                        # NaN in channel 0 (wins the arg-max)
    x[90:100, rng.integers(1, Cn, 10)] = np.nan                 # NaN in a later channel (skipped)
    x[100:110, rng.integers(0, Cn, 10)] = np.inf
    x[110:120, rng.integers(0, Cn, 10)] = -np.inf
    x[120:125] = -np.inf                                        # every value -inf
    x[125:130, :] = 7.0                                         # all equal
    x[130:140, rng.integers(0, Cn, 10)] = 60.0                  # one dominant class: p rounds to 1
    x[140:150] = np.float32(3e38) * np.sign(x[140:150])         # near the fp32 range
    return x


@pytest.mark.parametrize("order", [0, 1, 2], ids=["sequential", "two_threads_per_row", "xpacked_lane_pairs"])
def test_running_softmax_helpers(emul, order):
    rng = np.random.default_rng(7 + order)
    for Cn in list(range(2, 21)) + [24, 31, 32, 33, 47, 48, 57, 63, 64]:
        x = _vectors(Cn, rng)
        cls, conf = _emulate(emul, x, order)
        assert np.array_equal(cls.astype(np.int64), ref_class(x)), Cn
        check_conf(conf, x)
        # the class without the confidence is the same
        cls0, _ = _emulate(emul, x, order, conf=False)
        assert np.array_equal(cls0, cls)


def test_merge_orders_agree_on_the_class(emul):
    rng = np.random.default_rng(3)
    x = _vectors(20, rng)
    classes = [_emulate(emul, x, o)[0] for o in range(3)]
    assert np.array_equal(classes[0], classes[1]) and np.array_equal(classes[0], classes[2])


# ---- plan creation without a GPU -----------------------------------------------------------------------------------
def _desc(impl, Cout=20, out1_mode=_lib.OUT1_CLASS_U16_CONF, out1=FAKE):
    d = _lib.ConvDesc()
    d.impl, d.dtype, d.n_src = impl, _lib.DTYPE_F32, 1
    d.src[0], d.src_C[0], d.src_cstride[0] = FAKE, 16, 16
    d.B, d.ID, d.IH, d.IW = 2, 4, 6, 32
    d.stride[:] = [1, 1, 1]
    d.omul[:] = [1, 1, 1]
    taps = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]
    d.n_taps = len(taps)
    for i, (a, b, c) in enumerate(taps):
        d.taps[i].src, d.taps[i].dz, d.taps[i].dy, d.taps[i].dx = 0, a, b, c
    d.weight, d.bias = FAKE, FAKE
    d.Cout, d.Cout_pad, d.Kpad = Cout, (Cout + 15) // 16 * 16, 16
    d.OD, d.OH, d.OW = 4, 6, 32
    d.ODf, d.OHf, d.OWf = 4, 6, 32
    d.out1_mode, d.out1, d.out1_C = out1_mode, out1, Cout
    return d


def _create(d):
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.occd_conv_plan_create(C.byref(d), C.byref(h))
    msg = L.occd_last_error().decode() if rc else ""     # the last error is only meaningful on failure
    if rc == 0:
        L.occd_conv_plan_destroy(h)
    return rc, msg


def _outcomes(mode):
    """(return code, message) of every class-map descriptor case of tests/test_class_map_host.py, in mode `mode`"""
    res = []
    for impl, Cout, kw in ((_lib.CONV_IMPL_SIMT, 20, {}), (_lib.CONV_IMPL_SIMT, 80, {}),
                           (_lib.CONV_IMPL_SIMT, 20, dict(out1=None)), (_lib.CONV_IMPL_SIMT, 20, dict(out1=FAKE + 1)),
                           (_lib.CONV_IMPL_SIMT, 65536, {}), (_lib.CONV_IMPL_TC, 300, {})):
        res.append(_create(_desc(impl, Cout, mode, **kw)))
    d = _desc(_lib.CONV_IMPL_SIMT, out1_mode=mode)
    d.out0, d.out0_cstride = FAKE, 32
    res.append(_create(d))
    d = _desc(_lib.CONV_IMPL_TC, out1_mode=mode)
    d.n_groups, d.group_tap0[0], d.group_tap0[1], d.group_tap0[2] = 2, 0, 9, 27
    d.omul[:] = [2, 2, 2]
    d.ODf, d.OHf, d.OWf = 8, 12, 64
    d.group_oadd[1][:] = [1, 1, 1]
    res.append(_create(d))
    for impl in (_lib.CONV_IMPL_TC, _lib.CONV_IMPL_HALO, _lib.CONV_IMPL_HALOX, _lib.CONV_IMPL_TCX):
        res.append(_create(_desc(impl, 20, mode)))        # accepted up to the tensor-map encode, or refused alike
    return res


def test_mode4_is_accepted_and_refused_where_mode3_is():
    _build.build()
    m3, m4 = _outcomes(_lib.OUT1_CLASS_U16), _outcomes(_lib.OUT1_CLASS_U16_CONF)
    assert m3 == m4
    assert m4[0][0] == 0 and m4[5][0] == _lib.ERR_UNSUPPORTED and "one N tile" in m4[5][1]
    assert m4[6][0] == _lib.ERR_UNSUPPORTED and "only output" in m4[6][1]
    assert m4[7][0] == _lib.ERR_UNSUPPORTED
    L = _lib.lib()
    h = C.c_void_p()
    assert L.occd_conv_plan_create(C.byref(_desc(_lib.CONV_IMPL_SIMT)), C.byref(h)) == 0
    try:
        lut = (C.c_int * 20)(*range(100, 120))
        assert L.occd_conv_plan_set_class_lut(h, lut, 20) == 0                  # the remap applies to mode 4 too
        assert L.occd_conv_plan_set_class_lut(h, lut, 19) == _lib.ERR_ARG
    finally:
        L.occd_conv_plan_destroy(h)


def test_argmax_classes_conf_validates_its_arguments():
    _build.build()
    L = _lib.lib()
    f = L.occd_argmax_classes_conf
    lut = (C.c_int * 80)(*range(80))
    assert f(None, FAKE, FAKE, 1, 20, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, None, FAKE, 1, 20, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, None, 1, 20, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, FAKE, 0, 20, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, FAKE, 1, 0, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, FAKE, 1, 65536, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, FAKE, 1, 20, 0, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE + 1, FAKE, 1, 20, 8, None, None) == _lib.ERR_ARG           # uint16 alignment
    assert f(FAKE, FAKE, FAKE + 1, 1, 20, 8, None, None) == _lib.ERR_ARG
    assert f(FAKE, FAKE, FAKE, 1, 80, 8, lut, None) == _lib.ERR_ARG                # a remap covers at most 64
    assert b"occd_argmax_classes_conf" in L.occd_last_error()


def test_engine_falls_back_to_logits_and_argmax_classes_conf(monkeypatch):
    """Plan.conv(out1_mode="classes_conf"): one conv launch where the kernel writes map and confidence; where plan
    creation refuses it, planar logits into a plan-owned buffer and occd_argmax_classes_conf"""
    from occdepth_b200.engine import ClassMapUnsupported, ConvOp, Plan
    _build.build()
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    out = torch.empty(2, 2, 4, 6, 32, dtype=torch.uint16)
    plan.conv(x, torch.randn(20, 16, 3, 3, 3), torch.randn(20), padding=1, out1=out, out1_mode="classes_conf",
              lut=list(range(20)), no_out0=True, name="cls")
    assert [op.name for op in plan.ops] == ["cls"] and plan.ops[0].desc.out1_mode == _lib.OUT1_CLASS_U16_CONF
    with pytest.raises(ClassMapUnsupported, match="one N tile"):
        ConvOp([x], [(0, 0, 0, 0)], [torch.randn(300, 16)], torch.randn(300), (4, 6, 32), out1=out,
               out1_mode="classes_conf", impl=_lib.CONV_IMPL_TC, name="wide")
    # the fallback, with the planar launch planned as SIMT (no driver is needed to plan it): a kernel that refuses the
    # map is stood in for by ConvOp raising ClassMapUnsupported for the class-map modes
    import occdepth_b200.engine as E
    real = E.ConvOp

    def refusing(*a, **kw):
        if kw.get("out1_mode") in E.CLASS_MODES:
            raise ClassMapUnsupported("refused")
        return real(*a, **kw)
    monkeypatch.setattr(E, "ConvOp", refusing)
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    plan.conv(x, torch.randn(20, 16, 3, 3, 3), torch.randn(20), padding=1, out1=out, out1_mode="classes_conf",
              no_out0=True, name="cls")
    assert [op.name for op in plan.ops] == ["cls", "occd_argmax_classes_conf"]
    assert plan.ops[0].desc.out1_mode == _lib.OUT1_F32_PLANAR


@pytest.mark.parametrize("cascade", [False, True])
def test_decoder_class_conf_plan(monkeypatch, cascade):
    """the KITTI decoder with confidence ends in the fused classifier writing uint16 [2, B, X, Y, Z]"""
    from occdepth_b200.engine import Plan
    from occdepth_b200.models.unet3d_kitti import UNet3D
    _build.build()
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    with contextlib.redirect_stdout(io.StringIO()):
        m = UNet3D(20, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=False, cascade_cls=cascade,
                   occluded_cls=True).eval()
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(1, 16, 16, 8, 16)
    with torch.no_grad():
        y = m.emit(plan, x, classes=True, lut=list(range(20)), confidence=True)
    assert y.dtype == torch.uint16 and tuple(y.shape) == (2, 1, 32, 32, 16)
    last = "head.conv_classes.b" if cascade else "head.conv_classes"
    assert plan.ops[-1].name == last and plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16_CONF


# ---- the model loader ------------------------------------------------------------------------------------------------
def _model_file(flags, classes_len):
    """tests/test_deploy_host.py's tiny well-formed file (a 1 x 1 x 2 output grid: a 4-byte map) with header flags
    `flags` and a class-map role of classes_len bytes"""
    from test_deploy_host import model_file
    data = bytearray(model_file())
    # header: magic, <9I> (flags is the 5th), <7I>, the pattern, <7d>, <2I>, the LUT, <d3I>, <3I>, G, <I>, roles
    struct.pack_into("<I", data, 8 + 4 * 4, flags)
    roles_at = 8 + 36 + 28 + 512 + 56 + 8 + 256 + 20 + 12 + 64 + 4
    k, off, n = struct.unpack_from("<iQQ", data, roles_at + 7 * 20)
    assert n == 4
    struct.pack_into("<iQQ", data, roles_at + 7 * 20, k, off, classes_len)
    # the role's buffer grows with it
    n_buf = struct.unpack_from("<4I", data, roles_at + 8 * 20)[0]
    body = roles_at + 8 * 20 + 16
    bk = body + 12 * k
    size, kind = struct.unpack_from("<QI", data, bk)
    struct.pack_into("<QI", data, bk, max(size, classes_len), kind)
    assert k < n_buf
    return bytes(data)


def _load(tmp_path, data):
    L = _lib.lib()
    p = tmp_path / "m.occd"
    p.write_bytes(data)
    h = C.c_void_p()
    rc = L.occd_model_load(str(p).encode(), C.byref(h))
    if rc == 0:
        L.occd_model_destroy(h)
    return rc, L.occd_last_error().decode()


def _passes_validation(rc, msg):
    return rc == 0 or (rc == _lib.ERR_CUDA and "cudaMalloc" in msg)


def test_loader_confidence_flag(tmp_path, monkeypatch):
    _build.build()
    monkeypatch.syspath_prepend(os.path.dirname(os.path.abspath(__file__)))
    assert _passes_validation(*_load(tmp_path, _model_file(0, 4)))
    assert _passes_validation(*_load(tmp_path, _model_file(4, 8)))          # map, then its confidence
    rc, msg = _load(tmp_path, _model_file(4, 4))                            # flag bit 2 with a one-map role
    assert rc == _lib.ERR_FORMAT and "class map" in msg, msg
    rc, msg = _load(tmp_path, _model_file(0, 8))                            # a two-map role without the flag
    assert rc == _lib.ERR_FORMAT and "class map" in msg, msg
    for bit in (8, 1 << 31):
        rc, msg = _load(tmp_path, _model_file(bit, 4))
        assert rc == _lib.ERR_FORMAT and "unknown header flag bits" in msg, msg


def test_run_frame_conf_checks_its_arguments():
    _build.build()
    L = _lib.lib()
    f = _lib.Frame()
    assert L.occd_model_run_frame_conf(None, C.byref(f), FAKE, FAKE, None) == _lib.ERR_ARG
    assert b"occd_model_run_frame_conf" in L.occd_last_error()
