"""CPU checks of the model-file runtime (occd_model_load, include/occdepth_b200.h): the loader validates a whole file
before it touches a device and refuses malformed ones with the right code and message; every launch entry point
the ctypes bindings declare is replayable; occd_flosp_camera_tables equals FlospDepth.camera_tables bit for bit."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib
from occdepth_b200.deploy import MAGIC

# entry points that are not launches (no stream): never recorded by deploy.export
NOT_REPLAYED = {"occd_abi_version", "occd_last_error", "occd_conv_plan_create", "occd_conv_plan_destroy",
                "occd_conv_plan_info", "occd_conv_plan_impl", "occd_conv_plan_schedule",
                "occd_conv_plan_set_class_lut", "occd_conv_debug_trace", "occd_model_load", "occd_model_info",
                "occd_model_run_frame", "occd_model_destroy", "occd_flosp_camera_tables"}


def _lib_built():
    _build.build()
    return _lib.lib()


def _arg(tag, *v):
    fmt = {"p": "<IQ", "h": "<I", "c": "<I", "i": "<i", "l": "<q", "f": "<f", "d": "<d", "n": "", "s": ""}[tag]
    return tag.encode() + (struct.pack(fmt, *v) if fmt else b"")


def _record(name, args):
    nm = name.encode()
    return struct.pack("<H", len(nm)) + nm + struct.pack("<I", len(args)) + b"".join(args)


def model_file(records=None, blobs=(), plans=(), fmt=_lib.MODEL_FORMAT_VERSION, abi=None, magic=MAGIC):
    """a tiny well-formed model file: one 1 x 2 x 2 image, a 1 x 1 x 2 grid, one buffer per staged role"""
    abi = _lib_built().occd_abi_version() if abi is None else abi
    roles_len = [2 * 2 * 8 * 4, 2 * 16, 2, 2 * 8, 0, 0, 0, 2 * 2]       # img pix fov pix_z depth cams sps classes
    bufs = [n for n in roles_len if n]
    roles, k = [], 0
    for n in roles_len:
        roles.append((k, 0, n) if n else (-1, 0, 0))
        k += 1 if n else 0
    if records is None:
        records = [_record("occd_planar_to_cl", [_arg("p", 0, 0), _arg("p", 0, 64), _arg("i", 0), _arg("l", 1),
                                                 _arg("i", 3), _arg("l", 4), _arg("i", 8), _arg("s")])]
    hdr = magic + struct.pack("<9I", fmt, abi, 0, 0, 0, 1, 2, 2, 2) + struct.pack("<7I", 1, 1, 2, 1, 1, 2, 1)
    hdr += np.zeros(128, "<i4").tobytes() + struct.pack("<7d", 0.4, 0, 0, 0, 0.4, 0.4, 0.8)
    hdr += struct.pack("<2I", 20, 0) + np.zeros(64, "<i4").tobytes() + struct.pack("<d3I", 0.0, 0, 0, 0)
    hdr += struct.pack("<3I", 0, 0, 0)                                  # FlospDepth's grid: none
    hdr += np.zeros(16, "<f4").tobytes() + struct.pack("<I", 8)
    hdr += b"".join(struct.pack("<iQQ", *r) for r in roles)
    hdr += struct.pack("<4I", len(bufs), len(blobs), len(plans), len(records))
    body = b"".join(struct.pack("<QI", n, 0) for n in bufs)
    for data, fix in blobs:
        body += struct.pack("<Q", len(data)) + data + struct.pack("<I", len(fix))
        body += b"".join(struct.pack("<QIQ", *f) for f in fix)
    body += b"".join(struct.pack("<IiI", *p) for p in plans)
    return hdr + body + b"".join(records)


def _load(tmp_path, data):
    L = _lib_built()
    p = tmp_path / "m.occd"
    p.write_bytes(data)
    h = C.c_void_p()
    rc = L.occd_model_load(str(p).encode(), C.byref(h))
    if rc == 0:
        L.occd_model_destroy(h)
    else:
        assert not h.value                          # nothing handed out on failure
    return rc, L.occd_last_error().decode()


def _passes_validation(rc, msg):
    """a valid file either loads (a GPU is present) or stops at the first CUDA call"""
    return rc == 0 or (rc == _lib.ERR_CUDA and "cudaMalloc" in msg)


def test_well_formed_file_passes_validation(tmp_path):
    rc, msg = _load(tmp_path, model_file())
    assert _passes_validation(rc, msg), (rc, msg)


@pytest.mark.parametrize("case,code,text", [
    ("magic", _lib.ERR_FORMAT, "magic"),
    ("format", _lib.ERR_UNSUPPORTED, "format version"),
    ("abi", _lib.ERR_UNSUPPORTED, "ABI version"),
    ("truncated", _lib.ERR_FORMAT, "truncated"),
    ("truncated_header", _lib.ERR_FORMAT, "truncated"),
    ("trailing", _lib.ERR_FORMAT, "trailing"),
    ("entry", _lib.ERR_FORMAT, "unknown entry point 'occd_no_such_kernel'"),
    ("arity", _lib.ERR_FORMAT, "arguments"),
    ("arg_type", _lib.ERR_FORMAT, "wrong type"),
    ("fixup_blob", _lib.ERR_FORMAT, "fix-up outside the blob"),
    ("fixup_buffer", _lib.ERR_FORMAT, "fix-up outside buffer"),
    ("fixup_buffer_id", _lib.ERR_FORMAT, "buffer id 9 out of range"),
    ("arg_buffer_id", _lib.ERR_FORMAT, "buffer id out of range"),
    ("arg_offset", _lib.ERR_FORMAT, "pointer outside its buffer"),
    ("plan_id", _lib.ERR_FORMAT, "convolution plan id out of range"),
    ("conv_desc", _lib.ERR_FORMAT, "bad descriptor"),
])
def test_loader_refuses(tmp_path, case, code, text):
    good = model_file()
    sfa = [_arg("h", 0), _arg("s")]
    data = {
        "magic": lambda: model_file(magic=b"OCCDMODX"),
        "format": lambda: model_file(fmt=_lib.MODEL_FORMAT_VERSION + 1),
        "abi": lambda: model_file(abi=_lib_built().occd_abi_version() + 1),
        "truncated": lambda: good[:-3],
        "truncated_header": lambda: good[:40],
        "trailing": lambda: good + b"\0",
        "entry": lambda: model_file([_record("occd_no_such_kernel", [_arg("s")])]),
        "arity": lambda: model_file([_record("occd_softmax_planar", [_arg("s")])]),
        "arg_type": lambda: model_file([_record("occd_conv_run", [_arg("i", 3), _arg("s")])]),
        "fixup_blob": lambda: model_file([_record("occd_sfa_lift_fwd", sfa)], blobs=[(bytes(16), [(12, 0, 0)])]),
        "fixup_buffer": lambda: model_file([_record("occd_sfa_lift_fwd", sfa)], blobs=[(bytes(16), [(0, 0, 128)])]),
        "fixup_buffer_id": lambda: model_file([_record("occd_sfa_lift_fwd", sfa)], blobs=[(bytes(16), [(0, 9, 0)])]),
        "arg_buffer_id": lambda: model_file([_record("occd_conv_run", [_arg("p", 5, 0), _arg("s")])]),
        "arg_offset": lambda: model_file([_record("occd_conv_run", [_arg("p", 0, 128), _arg("s")])]),
        "plan_id": lambda: model_file([_record("occd_conv_run", [_arg("c", 0), _arg("s")])]),
        "conv_desc": lambda: model_file([_record("occd_conv_run", [_arg("c", 0), _arg("s")])],
                                        blobs=[(bytes(16), [])], plans=[(0, -1, 0)]),
    }[case]()
    rc, msg = _load(tmp_path, data)
    assert rc == code, (rc, msg)
    assert text in msg, msg


def test_missing_file(tmp_path):
    L = _lib_built()
    h = C.c_void_p()
    assert L.occd_model_load(str(tmp_path / "absent.occd").encode(), C.byref(h)) == _lib.ERR_IO
    assert b"cannot open" in L.occd_last_error() and not h.value


def test_every_launch_entry_point_is_replayable(tmp_path):
    """a record of each launch entry point, typed from _lib.SYMBOLS as deploy.export types it, passes validation:
    the runtime's table covers the bindings with the same parameter types"""
    cls = {C.c_int: ("i", 1), C.c_longlong: ("l", 1), C.c_float: ("f", 1.0), C.c_double: ("d", 1.0)}
    names = [n for n in _lib.SYMBOLS if n not in NOT_REPLAYED]
    assert len(names) >= 30
    for name in names:
        args = []
        for t in _lib.SYMBOLS[name][1]:
            args.append(_arg(*cls[t]) if t in cls else _arg("n"))
        rc, msg = _load(tmp_path, model_file([_record(name, args)]))
        assert _passes_validation(rc, msg), (name, rc, msg)


# ---- occd_flosp_camera_tables against FlospDepth.camera_tables ---------------------------------------------------------
def _flosp(dataset, ps):
    from occdepth_b200.models.flosp_depth.flosp_depth import FlospDepth, flosp_depth_conf_map
    conf = dict(flosp_depth_conf_map[dataset])
    scene = (60, 36, 60) if dataset == "NYU" else (256, 256, 32)
    conf.update(scene_size=scene, project_scale=ps, return_depth=False,
                depth_net_conf=dict(in_channels=8, mid_channels=8))
    return FlospDepth(**conf)


def _c_tables(cam_k, T, G, origin, ps, f32):
    L = _lib_built()
    n = cam_k.shape[0]
    dt = np.float32 if f32 else np.float64
    k = np.ascontiguousarray(cam_k, dt)
    t = np.ascontiguousarray(T, dt)
    cams = np.zeros((n, 40), np.float32)
    sps = np.zeros(n, np.float32)
    vn = np.zeros(3, np.int32)
    g = None if G is None else np.ascontiguousarray(G, np.float32)
    o = None if origin is None else np.ascontiguousarray(origin, np.float64)
    rc = L.occd_flosp_camera_tables(n, k.ctypes.data, t.ctypes.data, 1 if f32 else 0,
                                    None if g is None else g.ctypes.data, None if o is None else o.ctypes.data, ps,
                                    cams.ctypes.data, sps.ctypes.data, vn.ctypes.data)
    assert rc == 0, L.occd_last_error()
    return cams, sps, vn


def _random_calib(rng, n):
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = rng.uniform(30, 4000, n), rng.uniform(30, 4000, n)
    K[:, 0, 2], K[:, 1, 2] = rng.uniform(-800, 2000, n), rng.uniform(-800, 2000, n)
    K[:, 0, 1] = np.where(rng.random(n) < 0.3, rng.normal(0, 3, n), 0)
    K[:, 2, 2] = 1
    T = rng.normal(size=(n, 4, 4)) * rng.uniform(0.01, 50, (n, 1, 1))
    T[:, 3] = [0, 0, 0, 1]
    return K, T


def _assert_bits(cams, sps, want_cams, want_sps):
    assert np.array_equal(cams.view(np.uint32), want_cams.numpy().reshape(cams.shape).view(np.uint32))
    assert np.array_equal(sps.view(np.uint32), want_sps.numpy().reshape(-1).view(np.uint32))


@pytest.mark.parametrize("f32", [False, True])
def test_camera_tables_kitti_bit_exact(f32):
    import synthetic
    fd = _flosp("kitti", 2)
    G = fd._grid_to_lidar(None)[0].numpy()
    tt = torch.float32 if f32 else torch.float64
    # the default calibration, then 10 000 seeded random intrinsics and poses as 5 000 stereo pairs
    K0, Ts = synthetic.kitti_calib(1220, 370)
    cases = [(np.stack([K0, K0]), np.stack([t.astype(np.float64) for t in Ts[:2]]))]
    rng = np.random.default_rng(1 + f32)
    K, T = _random_calib(rng, 10000)
    cases += [(K[i:i + 2], T[i:i + 2]) for i in range(0, 10000, 2)]
    ks = [torch.from_numpy(k).to(tt) for k, _ in cases]
    ts = [torch.from_numpy(t).to(tt) for _, t in cases]
    ida = [torch.eye(4).unsqueeze(0).repeat(2, 1, 1)] * len(cases)
    want_cams, want_sps, _ = fd.camera_tables(ks, ts, ida, None, 2)
    got = [_c_tables(k.numpy(), t.numpy(), G, None, 2, f32) for k, t in zip(ks, ts)]
    _assert_bits(np.stack([g[0] for g in got]), np.concatenate([g[1] for g in got]), want_cams, want_sps)


@pytest.mark.parametrize("f32", [False, True])
def test_camera_tables_nyu_bit_exact(f32):
    fd = _flosp("NYU", 1)
    tt = torch.float32 if f32 else torch.float64
    rng = np.random.default_rng(7 + f32)
    origins = [np.array([-2.0, 0.5, -0.1]), np.zeros(3)] + [rng.uniform(-5, 5, 3) for _ in range(198)]
    K, T = _random_calib(rng, 10000)
    K[:50] = [[518.8579, 0, 320], [0, 518.8579, 240], [0, 0, 1]]       # the dataset's intrinsics
    n = 0
    for o in origins:
        ks = [torch.from_numpy(K[n + i:n + i + 1]).to(tt) for i in range(50)]
        ts = [torch.from_numpy(T[n + i:n + i + 1]).to(tt) for i in range(50)]
        n += 50
        want_cams, want_sps, vn = fd.camera_tables(ks, ts, [torch.eye(4)[None]] * 50, torch.from_numpy(o)[None], 1)
        got = [_c_tables(k.numpy(), t.numpy(), None, o, 1, f32) for k, t in zip(ks, ts)]
        _assert_bits(np.stack([g[0] for g in got]), np.concatenate([g[1] for g in got]), want_cams, want_sps)
        assert all(list(g[2]) == list(vn) for g in got)
    assert n == 10000
