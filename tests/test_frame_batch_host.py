"""CPU checks of batched camera frames: the argument checks of occd_virtual_view_items_fwd and occd_model_run_frames,
the refusals and per-frame consistency checks of OccDepth.predict_frames and CameraPipeline(batch=) that need no
device, the loader's validation of batched model files (header flag bit 5 and the batch block), records of the new
entry points accepted by the model-file replay table, and the export's recorder forwarding destructors."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200.deploy import MAGIC


def _lib_built():
    _build.build()
    return _lib.lib()


# ---- occd_virtual_view_items_fwd ------------------------------------------------------------------------------------
def _vv(L, depth_stride, dh=4, dw=5, **k):
    a = dict(in_=C.c_void_p(16), out=C.c_void_p(16), depth=C.c_void_p(16), dtype=_lib.DTYPE_F32, B=2, h=3, w=3, Cn=8,
             cs_in=8, cs_out=8)
    a.update(k)
    return L.occd_virtual_view_items_fwd(a["in_"], a["out"], a["depth"], a["dtype"], a["B"], a["h"], a["w"], a["Cn"],
                                         a["cs_in"], a["cs_out"], dh, dw, 1.0, depth_stride, None)


def test_virtual_view_items_argument_checks():
    L = _lib_built()
    assert _vv(L, -1) == _lib.ERR_ARG
    assert b"depth_stride" in L.occd_last_error()
    assert _vv(L, 4 * 5 - 1) == _lib.ERR_ARG                # non-zero and smaller than dh * dw
    assert b"depth_stride" in L.occd_last_error()
    # the checks occd_virtual_view_fwd makes, kept
    assert _vv(L, 0, depth=None) == _lib.ERR_ARG
    assert _vv(L, 20, B=0) == _lib.ERR_ARG
    assert _vv(L, 20, cs_in=12) == _lib.ERR_ARG
    assert _vv(L, 20, Cn=16) == _lib.ERR_ARG                # channel window wider than the strides
    assert b"channel window" in L.occd_last_error()
    assert _vv(L, 0, dtype=7) == _lib.ERR_ARG               # past the argument checks: the dtype dispatch refuses


def test_model_run_frames_and_batch_argument_checks():
    L = _lib_built()
    f = _lib.Frame()
    out = C.c_int(0)
    assert L.occd_model_batch(None, C.byref(out)) == _lib.ERR_ARG
    assert L.occd_model_run_frames(None, C.byref(f), 1, None, None, None) == _lib.ERR_ARG
    assert b"occd_model_run_frames" in L.occd_last_error()


# ---- predict_frames / CameraPipeline(batch=) refusals ------------------------------------------------------------------
def _model(name, **k):
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if os.path.join(root, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(root, "tools"))
    import shipped_configs
    if name in shipped_configs.CONFIGS:
        hw, full = ((96, 128), None) if shipped_configs.CONFIGS[name]["dataset"] == "NYU" else ((96, 320), (64, 64, 16))
        m, _, _ = shipped_configs.make_case(name, img_hw=hw, full=full, **k)
    else:
        m, _, _ = shipped_configs.make_case(spec=k.pop("spec"), **k)
    return m


def _kitti(V=2, H=96, W=320, **extra):
    f = {"img": np.zeros((V, H, W, 3), np.uint8), "cam_k": np.stack([np.eye(3)] * V),
         "T_velo_2_cam": np.stack([np.eye(4)] * V), "img_hw": (H, W)}
    f.update(extra)
    return f


@pytest.fixture(scope="module")
def kitti_model():
    return _model("kitti_b3_f32_flospdepth_2080ti")


def test_predict_frames_refusals(kitti_model):
    m = kitti_model
    with pytest.raises(TypeError, match="list of frame dicts"):
        m.predict_frames(_kitti())
    with pytest.raises(ValueError, match="0 frames"):
        m.predict_frames([])
    with pytest.raises(ValueError, match="confidence=True"):
        m.predict_frames([_kitti()], classes=False, confidence=True)
    from occdepth_b200.parallel import SimSlabGroup
    m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
    try:
        with pytest.raises(NotImplementedError, match="one frame per forward"):
            m.predict_frames([_kitti(), _kitti()])
    finally:
        m.__dict__.pop("slab_ctx", None)


def test_predict_frames_refuses_infer_mode_flosp_depth():
    m = _model("kitti_b3_f32_flospdepth_2080ti", infer_mode=True)
    with pytest.raises(NotImplementedError, match="infer_mode with flosp_depth"):
        m.predict_frames([_kitti(), _kitti()])


def test_predict_frames_refuses_nyu_flosp_depth_batches():
    spec = dict(dataset="NYU", backbone_2d_name="tf_efficientnet_b3_ns", feature=16, trans_2d_to_3d="flosp_depth",
                views=1, context_prior=False, cascade_cls=False, use_depth_gt=True)
    m = _model(None, spec=spec)
    frame = {"img": np.zeros((480, 640, 3), np.uint8), "cam_pose": np.eye(4), "vox_origin": np.zeros(3)}
    with pytest.raises(NotImplementedError, match="FlospDepth prior"):
        m.predict_frames([frame, frame])


@pytest.mark.parametrize("key,frame1", [
    ("V", _kitti(V=1)),
    ("img_hw", _kitti(img_hw=(96, 288))),
    ("voxel_size", _kitti(voxel_size=0.2)),
    ("scene_size", _kitti(scene_size=(25.6, 25.6, 3.2))),
    ("pattern_id", _kitti(pattern_id=1)),
    ("depth", _kitti(depth=np.zeros((96, 320), np.uint16))),
])
def test_predict_frames_frames_must_agree(kitti_model, key, frame1):
    with pytest.raises(ValueError, match="frame 1's %s" % key):
        kitti_model.predict_frames([_kitti(), frame1])


def test_predict_frames_frames_may_differ_in_calibration_and_raw_size(kitti_model):
    """what may differ passes the host checks (and stops at the device check on a machine without one)"""
    other = _kitti(H=100, W=330, cam_k=np.stack([np.eye(3) * 2] * 2), vox_origin=np.array([0.0, -12.8, -2.0]))
    other["img_hw"] = (96, 320)
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the full run is the GPU suite's")
    with pytest.raises(RuntimeError):
        kitti_model.predict_frames([_kitti(), other])


def test_camera_pipeline_batch_refusals(kitti_model):
    from occdepth_b200.serving import CameraPipeline
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="batch must be"):
            CameraPipeline(kitti_model, img_hw=(96, 320), batch=bad)
    with pytest.raises(ValueError, match="output='voxels'"):
        CameraPipeline(kitti_model, img_hw=(96, 320), batch=2, output="voxels")
    with pytest.raises(ValueError, match="slab_output"):
        CameraPipeline(kitti_model, img_hw=(96, 320), batch=2, slab_output="slab")


def test_export_of_a_batch_refuses_slab_output(kitti_model, tmp_path):
    with pytest.raises(NotImplementedError, match="no X-slab partition"):
        deploy.export(kitti_model, tmp_path / "x.occd", [_kitti(), _kitti()], slab_output="root")
    assert not (tmp_path / "x.occd").exists()


# ---- batched model files: the loader ----------------------------------------------------------------------------------
def _arg(tag, *v):
    fmt = {"p": "<IQ", "h": "<I", "c": "<I", "i": "<i", "l": "<q", "f": "<f", "d": "<d", "n": "", "s": ""}[tag]
    return tag.encode() + (struct.pack(fmt, *v) if fmt else b"")


def _record(name, args):
    nm = name.encode()
    return struct.pack("<H", len(nm)) + nm + struct.pack("<I", len(args)) + b"".join(args)


def batch_file(B=2, block=True, flags=deploy.FLAG_BATCH, role_items=None, records=None, slab_block=False):
    """a tiny batched model file: B items of one 1 x 2 x 2 image and a 1 x 1 x 2 grid, one buffer per staged role.
    role_items: the item count the roles are sized for (default B); block: whether the batch block is written"""
    abi = _lib_built().occd_abi_version()
    items = B if role_items is None else role_items
    per_item = [2 * 2 * 8 * 4, 2 * 16, 2, 2 * 8, 0, 0, 0, 2 * 2]      # img pix fov pix_z depth cams sps classes
    bufs = [n * items for n in per_item if n]
    roles, k = [], 0
    for n in per_item:
        roles.append((k, 0, n * items) if n else (-1, 0, 0))
        k += 1 if n else 0
    if records is None:
        records = [_record("occd_planar_to_cl", [_arg("p", 0, 0), _arg("p", 0, 64), _arg("i", 0), _arg("l", 1),
                                                 _arg("i", 3), _arg("l", 4), _arg("i", 8), _arg("s")])]
    hdr = MAGIC + struct.pack("<9I", _lib.MODEL_FORMAT_VERSION, abi, 0, 0, flags, 1, 2, 2, 2)
    hdr += struct.pack("<7I", 1, 1, 2, 1, 1, 2, 1)
    hdr += np.zeros(128, "<i4").tobytes() + struct.pack("<7d", 0.4, 0, 0, 0, 0.4, 0.4, 0.8)
    hdr += struct.pack("<2I", 20, 0) + np.zeros(64, "<i4").tobytes() + struct.pack("<d3I", 0.0, 0, 0, 0)
    hdr += struct.pack("<3I", 0, 0, 0) + np.zeros(16, "<f4").tobytes() + struct.pack("<I", 8)
    hdr += b"".join(struct.pack("<iQQ", *r) for r in roles)
    if block:
        hdr += struct.pack("<I", B)
    if slab_block:                                # rank 0 of 1, bounds [0, 1), the whole window, every view, map X 1
        hdr += struct.pack("<2I", 0, 1) + struct.pack("<2I", 0, 1) + struct.pack("<2QiI", 0, 2, -1, 1)
    hdr += struct.pack("<4I", len(bufs), 0, 0, len(records))
    body = b"".join(struct.pack("<QI", n, 0) for n in bufs)
    return hdr + body + b"".join(records)


def _load(tmp_path, data):
    L = _lib_built()
    p = tmp_path / "m.occd"
    p.write_bytes(data)
    h = C.c_void_p()
    rc = L.occd_model_load(str(p).encode(), C.byref(h))
    if rc == 0:
        b = C.c_int(0)
        assert L.occd_model_batch(h, C.byref(b)) == 0
        L.occd_model_destroy(h)
        return rc, "", b.value
    assert not h.value
    return rc, L.occd_last_error().decode(), None


def _passes_validation(rc, msg):
    """a valid file either loads (a GPU is present) or stops at the first CUDA call"""
    return rc == 0 or (rc == _lib.ERR_CUDA and "cudaMalloc" in msg)


@pytest.mark.parametrize("B", [1, 2, 3])
def test_well_formed_batched_file_passes_validation(tmp_path, B):
    rc, msg, b = _load(tmp_path, batch_file(B))
    assert _passes_validation(rc, msg), (rc, msg)
    if rc == 0:
        assert b == B


@pytest.mark.parametrize("case,text", [
    ("bit5_without_block", None),
    ("batch_zero", "out of range"),
    ("roles_not_B_items", "does not match the header"),
    ("roles_one_item", "does not match the header"),
    ("bits4_and_5", "flag bits 4 and 5"),
    ("block_without_bit5", None),
])
def test_loader_refuses_malformed_batched_files(tmp_path, case, text):
    data = {"bit5_without_block": lambda: batch_file(2, block=False),
            "batch_zero": lambda: batch_file(0, role_items=1),
            "roles_not_B_items": lambda: batch_file(3, role_items=2),
            "roles_one_item": lambda: batch_file(2, role_items=1),
            "bits4_and_5": lambda: batch_file(1, flags=deploy.FLAG_BATCH | deploy.FLAG_SLAB, slab_block=True),
            "block_without_bit5": lambda: batch_file(2, flags=0, role_items=1)}[case]()
    rc, msg, _ = _load(tmp_path, data)
    assert rc == _lib.ERR_FORMAT, (rc, msg)
    if text:
        assert text in msg, msg


def test_new_entry_points_are_replayable(tmp_path):
    """records of occd_virtual_view_items_fwd and occd_model_run_frames, typed from _lib.SYMBOLS as deploy.export types
    them, pass the loader's validation (the model handle of a recorded occd_model_run_frames can only be NULL)"""
    cls = {C.c_int: ("i", 1), C.c_longlong: ("l", 1), C.c_float: ("f", 1.0), C.c_double: ("d", 1.0)}
    for name in ("occd_virtual_view_items_fwd", "occd_model_run_frames"):
        args = [_arg(*cls[t]) if t in cls else _arg("n") for t in _lib.SYMBOLS[name][1]]
        rc, msg, _ = _load(tmp_path, batch_file(2, records=[_record(name, args)]))
        assert _passes_validation(rc, msg), (name, rc, msg)
    # a buffer pointer in the model-handle slot of occd_model_run_frames is refused
    args = [_arg("p", 0, 0), _arg("n"), _arg("i", 1), _arg("n"), _arg("n"), _arg("s")]
    rc, msg, _ = _load(tmp_path, batch_file(2, records=[_record("occd_model_run_frames", args)]))
    assert rc == _lib.ERR_FORMAT and "wrong type" in msg, msg


def test_recorder_forwards_destructors_while_recording():
    """a plan or model that the garbage collector finalizes on the exporting thread during the recording run is
    released through the library, not recorded into the file (a handle is no pointer into the plan's buffers)"""
    class Fake:
        def __init__(self):
            self.released = []

        def occd_conv_plan_destroy(self, h):
            self.released.append(("plan", h.value))
            return 0

        def occd_model_destroy(self, h):
            self.released.append(("model", h.value))
            return 0

    fake = Fake()
    rec = deploy._Recorder(fake)
    rec.recording = True
    assert rec.occd_conv_plan_destroy(C.c_void_p(0x1230)) == 0
    assert rec.occd_model_destroy(C.c_void_p(0x4560)) == 0
    assert rec.calls == []
    assert fake.released == [("plan", 0x1230), ("model", 0x4560)]
