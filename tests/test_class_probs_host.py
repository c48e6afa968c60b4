"""Class probabilities (OCCD_OUT1_CLASS_U16_PROBS) on the host.

- The class-map epilogues' running softmax and their second, probability-writing pass (ClassArg and class_arg_prob,
  csrc/conv_common.cuh), compiled for the CPU (tests/host_emul/class_probs_emul.cu) and driven in each epilogue's merge
  order: every probability is float16(p) or a float16 neighbour of it, p the float64 softmax; NaN in every class
  exactly where a logit is NaN or +inf (or all are -inf); the probability at the map's class is mode 4's confidence,
  bit for bit.
- Plan creation without a GPU: mode 5 is accepted and refused where mode 3 is, occd_class_probs checks its arguments,
  and the engine falls back to logits + occd_class_probs.
- The Python refusals of probabilities=True."""
import contextlib
import ctypes as C
import io
import os
import shutil
import subprocess

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
    out = tmp_path_factory.mktemp("class_probs_emul") / "libclass_probs_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "class_probs_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).class_probs_emulate
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def _emulate(fn, x, order):
    x = np.ascontiguousarray(x, np.float32)
    n, Cn = x.shape
    cls = np.zeros(n, np.uint16)
    conf = np.zeros(n, np.uint16)
    probs = np.zeros((n, Cn), np.uint16)
    assert fn(x.ctypes.data, n, Cn, order, cls.ctypes.data, conf.ctypes.data, probs.ctypes.data) == 0
    return cls, conf, probs


def _vectors(Cn, rng, n=400):
    x = rng.normal(0, 3, (n, Cn)).astype(np.float32)
    x[:40] = np.round(x[:40])                                  # ties
    x[40:60] = x[40:60] * 1e-4                                  # near-uniform
    x[60:80] *= 1e29                                            # magnitudes of about 1e30
    x[80:90, 0] = np.nan                                        # NaN in channel 0
    x[90:100, rng.integers(1, Cn, 10)] = np.nan                 # NaN in a later channel
    x[100:110, rng.integers(0, Cn, 10)] = np.inf
    x[110:120, rng.integers(0, Cn, 10)] = -np.inf               # one class impossible: probability 0
    x[120:125] = -np.inf                                        # every value -inf
    x[125:130, :] = 7.0                                         # all equal
    x[130:140, rng.integers(0, Cn, 10)] = 60.0                  # one dominant class
    x[140:150] = np.float32(3e38) * np.sign(x[140:150])         # near the fp32 range
    x[150:160] = rng.normal(0, 30, (10, Cn))                    # probabilities below float16's normal range
    return x


def check_probs(probs, logits):
    """probs (float16 bits [n, C]) against the float64 softmax of logits: float16(p) or a float16 neighbour of it
    (a one-ulp band), NaN exactly where p is NaN"""
    p = torch.softmax(torch.as_tensor(np.asarray(logits, np.float64)), dim=1).numpy()
    got = probs.view(np.float16)
    nan_p = np.isnan(p)
    assert np.array_equal(np.isnan(got), nan_p), np.argwhere(np.isnan(got) != nan_p)[:10]
    h = p[~nan_p].astype(np.float16)
    g = got[~nan_p]
    ok = (g == h) | (g == np.nextafter(h, np.float16(np.inf))) | (g == np.nextafter(h, np.float16(-np.inf)))
    assert ok.all(), list(zip(g[~ok][:5], p[~nan_p][~ok][:5]))


@pytest.mark.parametrize("order", [0, 1, 2], ids=["sequential", "two_threads_per_row", "xpacked_lane_pairs"])
def test_probabilities_against_float64_softmax(emul, order):
    rng = np.random.default_rng(11 + order)
    for Cn in list(range(2, 21)) + [24, 31, 32, 33, 47, 48, 64, 80, 96]:
        x = _vectors(Cn, rng)
        cls, conf, probs = _emulate(emul, x, order)
        check_probs(probs, x)
        # a NaN or +inf logit, or all -inf, makes every class of the voxel NaN, as torch.softmax does
        bad = np.isnan(x).any(1) | np.isposinf(x).any(1) | np.isneginf(x).all(1)
        assert np.isnan(probs.view(np.float16)[bad]).all()
        assert not np.isnan(probs.view(np.float16)[~bad]).any()


@pytest.mark.parametrize("order", [0, 1, 2], ids=["sequential", "two_threads_per_row", "xpacked_lane_pairs"])
def test_top_class_probability_is_the_confidence(emul, order):
    rng = np.random.default_rng(5 + order)
    for Cn in (2, 12, 20, 33, 64):
        x = _vectors(Cn, rng)
        cls, conf, probs = _emulate(emul, x, order)
        top = probs[np.arange(len(x)), cls.astype(np.int64)]
        assert np.array_equal(top, conf), Cn


def test_probabilities_leave_the_class_alone(emul):
    """mode 5's class is mode 3's: the first index of the largest value, whatever the merge order"""
    rng = np.random.default_rng(3)
    x = _vectors(20, rng)
    classes = [_emulate(emul, x, o)[0] for o in range(3)]
    ref = np.zeros(len(x), np.int64)
    for i, v in enumerate(x):
        if not np.isnan(v[0]):
            ref[i] = int(np.argmax(np.where(np.isnan(v), -np.inf, v.astype(np.float64))))
    for c in classes:
        assert np.array_equal(c.astype(np.int64), ref)


# ---- plan creation without a GPU -----------------------------------------------------------------------------------
def test_mode5_is_accepted_and_refused_where_mode3_is(monkeypatch):
    monkeypatch.syspath_prepend(os.path.dirname(os.path.abspath(__file__)))
    from test_class_conf_host import _desc, _outcomes
    _build.build()
    m3, m5 = _outcomes(_lib.OUT1_CLASS_U16), _outcomes(_lib.OUT1_CLASS_U16_PROBS)
    assert m3 == m5
    assert m5[0][0] == 0 and m5[5][0] == _lib.ERR_UNSUPPORTED and "one N tile" in m5[5][1]
    L = _lib.lib()
    h = C.c_void_p()
    assert L.occd_conv_plan_create(C.byref(_desc(_lib.CONV_IMPL_SIMT, out1_mode=_lib.OUT1_CLASS_U16_PROBS)),
                                   C.byref(h)) == 0
    try:
        lut = (C.c_int * 20)(*range(100, 120))
        assert L.occd_conv_plan_set_class_lut(h, lut, 20) == 0
    finally:
        L.occd_conv_plan_destroy(h)


def test_class_probs_validates_its_arguments():
    _build.build()
    L = _lib.lib()
    f = L.occd_class_probs
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
    assert b"occd_class_probs" in L.occd_last_error()


def test_engine_falls_back_to_logits_and_class_probs(monkeypatch):
    from occdepth_b200.engine import ClassMapUnsupported, Plan
    import occdepth_b200.engine as E
    _build.build()
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    out = torch.empty(21 * 2, 4, 6, 32, dtype=torch.uint16)
    plan.conv(x, torch.randn(20, 16, 3, 3, 3), torch.randn(20), padding=1, out1=out, out1_mode="classes_probs",
              lut=list(range(20)), no_out0=True, name="cls")
    assert [op.name for op in plan.ops] == ["cls"] and plan.ops[0].desc.out1_mode == _lib.OUT1_CLASS_U16_PROBS
    real = E.ConvOp

    def refusing(*a, **kw):
        if kw.get("out1_mode") in E.CLASS_MODES:
            raise ClassMapUnsupported("refused")
        return real(*a, **kw)
    monkeypatch.setattr(E, "ConvOp", refusing)
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(2, 4, 6, 32, 16)
    plan.conv(x, torch.randn(20, 16, 3, 3, 3), torch.randn(20), padding=1, out1=out, out1_mode="classes_probs",
              no_out0=True, name="cls")
    assert [op.name for op in plan.ops] == ["cls", "occd_class_probs"]
    assert plan.ops[0].desc.out1_mode == _lib.OUT1_F32_PLANAR


@pytest.mark.parametrize("cascade", [False, True])
def test_decoder_class_probs_plan(monkeypatch, cascade):
    """the KITTI decoder with probabilities ends in the fused classifier writing the map and the probabilities"""
    from occdepth_b200.engine import Plan
    from occdepth_b200.models.modules import split_probs
    from occdepth_b200.models.unet3d_kitti import UNet3D
    _build.build()
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    with contextlib.redirect_stdout(io.StringIO()):
        m = UNet3D(20, nn.BatchNorm3d, (32, 32, 16), 16, 2, context_prior=False, cascade_cls=cascade,
                   occluded_cls=True).eval()
    plan = Plan(torch.device("cpu"), precision="tf32")
    x = plan.alloc(1, 16, 16, 8, 16)
    with torch.no_grad():
        y = m.emit(plan, x, classes=True, lut=list(range(20)), probabilities=True)
    assert y.dtype == torch.uint16 and tuple(y.shape) == (21, 32, 32, 16)
    cmap, probs = split_probs(y, 1)
    assert tuple(cmap.shape) == (1, 32, 32, 16) and cmap.data_ptr() == y.data_ptr()
    assert probs.dtype == torch.float16 and tuple(probs.shape) == (1, 20, 32, 32, 16)
    assert probs.data_ptr() == y.data_ptr() + 2 * 32 * 32 * 16
    last = "head.conv_classes.b" if cascade else "head.conv_classes"
    assert plan.ops[-1].name == last and plan.ops[-1].desc.out1_mode == _lib.OUT1_CLASS_U16_PROBS


def test_probabilities_refusals():
    from occdepth_b200.models.OccDepth import OccDepth
    x = torch.zeros(1, 20, 2, 2, 2)
    with pytest.raises(ValueError, match="already hold the confidence"):
        OccDepth.class_map(x, confidence=True, probabilities=True)
    m = OccDepth.__new__(OccDepth)
    nn.Module.__init__(m)
    with pytest.raises(ValueError, match="already hold the confidence"):
        m.predict_classes({}, confidence=True, probabilities=True)
    with pytest.raises(ValueError, match=r"class map's probabilities \(classes=True\)"):
        m.predict_frame({}, classes=False, probabilities=True)
    with pytest.raises(ValueError, match="already hold the confidence"):
        m.predict_frame({}, confidence=True, probabilities=True)
    with pytest.raises(ValueError, match=r"class map's probabilities \(classes=True\)"):
        m.predict_frames([{}], classes=False, probabilities=True)
    with pytest.raises(ValueError, match="already hold the confidence"):
        m.predict_frames([{}], confidence=True, probabilities=True)


def test_mode5_refuses_wide_row_tiles_where_mode3_takes_them(monkeypatch):
    """97 to 128 classes on a grid large enough for one N tile of 112 or 128 channels: mode 3 gets past the tile
    choice (planned, or on a host without a driver stopped at the tensor-map encode), mode 5 is refused (the engine
    then falls back to logits + occd_class_probs); at 96 classes both are planned alike"""
    monkeypatch.syspath_prepend(os.path.dirname(os.path.abspath(__file__)))
    import test_class_conf_host as T
    _build.build()

    def create(Cout, mode, dtype):
        d = T._desc(_lib.CONV_IMPL_TC, Cout, mode)
        d.dtype = dtype
        d.B, d.ID, d.IH, d.IW = 2, 16, 64, 64
        d.OD, d.OH, d.OW = d.ODf, d.OHf, d.OWf = 16, 64, 64
        return T._create(d)
    for dtype in (_lib.DTYPE_F32, _lib.DTYPE_BF16):
        assert create(96, _lib.OUT1_CLASS_U16, dtype) == create(96, _lib.OUT1_CLASS_U16_PROBS, dtype)
        for Cout in (97, 112, 128):
            m3, m5 = create(Cout, _lib.OUT1_CLASS_U16, dtype), create(Cout, _lib.OUT1_CLASS_U16_PROBS, dtype)
            assert m3[0] == 0 or "one N tile" not in m3[1], (Cout, m3)
            assert m5[0] == _lib.ERR_UNSUPPORTED and "at most 96" in m5[1], (Cout, m5)


# ---- the model loader ------------------------------------------------------------------------------------------------
N_CLASSES_AT = 8 + 36 + 28 + 512 + 56      # header: magic, <9I>, <7I>, the pattern, <7d>, then n_classes


def test_loader_probabilities_flag(tmp_path, monkeypatch):
    import struct
    monkeypatch.syspath_prepend(os.path.dirname(os.path.abspath(__file__)))
    from test_class_conf_host import _load, _model_file, _passes_validation
    _build.build()
    n_classes = struct.unpack_from("<I", _model_file(0, 4), N_CLASSES_AT)[0]
    assert n_classes >= 1
    assert _passes_validation(*_load(tmp_path, _model_file(256, 4 * (1 + n_classes))))   # map, then C planes
    for length in (4, 8, 4 * n_classes, 4 * (2 + n_classes)):
        rc, msg = _load(tmp_path, _model_file(256, length))
        assert rc == _lib.ERR_FORMAT and "class map" in msg, (length, msg)
    rc, msg = _load(tmp_path, _model_file(256 | 4, 4 * (1 + n_classes)))
    assert rc == _lib.ERR_FORMAT and "together" in msg, msg
    for bit in (8, 128, 1 << 31):                                          # still unknown
        rc, msg = _load(tmp_path, _model_file(bit, 4))
        assert rc == _lib.ERR_FORMAT and "unknown header flag bits" in msg, msg


def test_run_frames_probs_checks_its_arguments():
    _build.build()
    L = _lib.lib()
    fx = (_lib.FrameEx * 1)()
    assert L.occd_model_run_frames_probs(None, fx, 1, FAKE, FAKE, None) == _lib.ERR_ARG
    assert b"occd_model_run_frames_probs" in L.occd_last_error()
    hs = (C.c_void_p * 1)(None)
    f = _lib.Frame()
    assert L.occd_model_run_frame_group_probs(hs, 1, C.byref(f), FAKE, None, None) == _lib.ERR_ARG
    assert L.occd_comm_gather_root_items(None, FAKE, FAKE, (C.c_int * 2)(0, 1), 8, 2, None) == _lib.ERR_ARG


def test_run_frames_probs_without_the_flag(tmp_path, monkeypatch):
    """a file exported without probabilities: the probabilities call is refused before anything runs"""
    monkeypatch.syspath_prepend(os.path.dirname(os.path.abspath(__file__)))
    from test_class_conf_host import _model_file
    _build.build()
    L = _lib.lib()
    p = tmp_path / "m.occd"
    p.write_bytes(_model_file(0, 4))
    h = C.c_void_p()
    rc = L.occd_model_load(str(p).encode(), C.byref(h))
    if rc != 0:
        pytest.skip("the loader needs a device past validation here: %s" % L.occd_last_error().decode())
    try:
        fx = (_lib.FrameEx * 1)()
        fx[0].frame.images = FAKE
        assert L.occd_model_run_frames_probs(h, fx, 1, FAKE, FAKE, None) == _lib.ERR_UNSUPPORTED
        assert b"without probabilities" in L.occd_last_error()
    finally:
        L.occd_model_destroy(h)
