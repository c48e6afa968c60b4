"""Camera formats on the host: the loader's checks of a model file's rectification maps (header flag bit 6 and the maps
role), records of the new entry points accepted by the replay table, and the frame checks of the Python routes."""
import struct

import numpy as np
import pytest
import torch

from occdepth_b200 import _lib, deploy
from occdepth_b200.deploy import MAGIC

from test_frame_batch_host import _arg, _kitti, _lib_built, _load, _passes_validation, _record, kitti_model  # noqa: F401


def maps_file(flags=deploy.FLAG_MAPS, maps_role="own", maps_len=32, records=None):
    """a tiny model file: one 1 x 2 x 2 image, a 1 x 1 x 2 grid, one buffer per staged role; with FLAG_MAPS a maps role
    follows the roles -- "own": a buffer of its own of maps_len bytes, "none": buffer -1, None: no role written"""
    abi = _lib_built().occd_abi_version()
    per = [2 * 2 * 8 * 4, 2 * 16, 2, 2 * 8, 0, 0, 0, 2 * 2]        # img pix fov pix_z depth cams sps classes
    bufs = [n for n in per if n]
    roles, k = [], 0
    for n in per:
        roles.append((k, 0, n) if n else (-1, 0, 0))
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
    if maps_role == "own":
        hdr += struct.pack("<iQQ", len(bufs), 0, maps_len)
        bufs.append(maps_len)
    elif maps_role == "none":
        hdr += struct.pack("<iQQ", -1, 0, 0)
    hdr += struct.pack("<4I", len(bufs), 0, 0, len(records))
    body = b"".join(struct.pack("<QI", n, 0) for n in bufs)
    return hdr + body + b"".join(records)


def test_file_with_maps_passes_validation(tmp_path):
    rc, msg, _ = _load(tmp_path, maps_file())
    assert _passes_validation(rc, msg), (rc, msg)


@pytest.mark.parametrize("kw,text", [
    (dict(maps_role="none"), "without a maps buffer"),
    (dict(maps_len=28), "rectification maps buffer does not match"),
    (dict(maps_len=64), "rectification maps buffer does not match"),
    (dict(maps_role=None), None),                    # the bit without the role: the next fields are misread
    (dict(flags=0), None),                           # a role without the bit: trailing bytes
    (dict(flags=128, maps_role=None), "unknown header flag bits"),
])
def test_loader_refuses_malformed_maps(tmp_path, kw, text):
    rc, msg, _ = _load(tmp_path, maps_file(**kw))
    assert rc == _lib.ERR_FORMAT, (kw, rc, msg)
    if text:
        assert text in msg, msg


def test_new_entry_points_are_replayable(tmp_path):
    """records of occd_stage_camera_u8_cl and occd_model_run_frames_ex, typed from _lib.SYMBOLS as deploy.export types
    them, pass the loader's validation (a recorded occd_model_run_frames_ex can only hold a NULL model)"""
    import ctypes as C
    cls = {C.c_int: ("i", 1), C.c_longlong: ("l", 1), C.c_float: ("f", 1.0), C.c_double: ("d", 1.0)}
    for name in ("occd_stage_camera_u8_cl", "occd_model_run_frames_ex"):
        args = [_arg(*cls[t]) if t in cls else _arg("n") for t in _lib.SYMBOLS[name][1]]
        rc, msg, _ = _load(tmp_path, maps_file(records=[_record(name, args)]))
        assert _passes_validation(rc, msg), (name, rc, msg)


def test_model_run_frames_ex_argument_checks():
    L = _lib_built()
    fx = (_lib.FrameEx * 1)()
    assert L.occd_model_run_frames_ex(None, fx, 1, None, None, None) == _lib.ERR_ARG
    assert L.occd_last_error() == b"occd_model_run_frames_ex: null argument"


def test_frame_checks(kitti_model):                   # noqa: F811
    m = kitti_model
    dev = torch.device("cpu")
    f = _kitti()
    with pytest.raises(ValueError, match="pixel_format"):
        m._frame_inputs(dict(f, pixel_format="yuyv"), dev)
    with pytest.raises(ValueError, match="NV12"):                  # 149 rows: no whole luma height
        m._frame_inputs(dict(f, pixel_format="nv12", img=np.zeros((2, 149, 326), np.uint8)), dev)
    with pytest.raises(ValueError, match="NV12"):                  # odd width
        m._frame_inputs(dict(f, pixel_format="nv12", img=np.zeros((2, 150, 325), np.uint8)), dev)
    with pytest.raises(ValueError, match="NV12"):                  # an RGB array
        m._frame_inputs(dict(f, pixel_format="nv12"), dev)
    H, W = f["img_hw"]
    with pytest.raises(ValueError, match="rect_maps"):
        m._frame_inputs(dict(f, rect_maps=np.zeros((2, 2, H, W + 1), np.float32)), dev)
    with pytest.raises(ValueError, match="rect_maps"):
        m._frame_inputs(dict(f, rect_maps=np.zeros((2, 2, H, W), np.float64)), dev)
    got = m._frame_inputs(dict(f, pixel_format="nv12", img=np.zeros((2, 150, 326), np.uint8),
                               rect_maps=np.zeros((2, 2, H, W), np.float32), voxel_size=0.4,
                               scene_size=(12.8, 12.8, 3.2)), dev)
    assert got["pixel_format"] == "nv12" and got["V"] == 2 and tuple(got["maps"].shape) == (2, 2, H, W)
    # every multiple of 3 rows is an even luma height, 2 mod 4 too: KITTI's raw 370 and 374 rows (555 and 561 array
    # rows), 98 rows (147)
    for rows in (555, 561, 147):
        got = m._frame_inputs(dict(f, pixel_format="nv12", img=np.zeros((2, rows, 1242), np.uint8),
                                   rect_maps=np.zeros((2, 2, H, W), np.float32), voxel_size=0.4,
                                   scene_size=(12.8, 12.8, 3.2)), dev)
        assert tuple(got["imgs"].shape) == (2, rows, 1242)
    one = m._frame_signature(dict(f, pixel_format="nv12", img=np.zeros((2, 150, 326), np.uint8)))
    assert one == m._frame_signature(f)                            # the same V either way


def test_staging_kernels_do_not_spill():
    """ptxas reports no spill for any instantiation of the staging kernel (3 formats x maps or not x 2 output types),
    from the log the build writes next to the object"""
    import os
    import re
    log = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "occdepth_b200", "lib", "obj",
                       "vox2pix.o.log")
    if not os.path.exists(log):
        pytest.skip("library not built (no ptxas log)")
    kernels, entry = {}, None
    for line in open(log):
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            entry = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and entry and "stage_camera_kernel" in entry:
            kernels[entry] = (int(m.group(1)), int(m.group(2)))
            entry = None
    assert len(kernels) == 12, sorted(kernels)
    assert all(v == (0, 0) for v in kernels.values()), kernels


def test_model_file_frames_are_checked_before_the_library_reads_them():
    """LoadedModel's frames: the format is the frame's unless the call sets it, a disagreeing frame and a frame with its
    own rect_maps are refused, and the images must be the model's V views of the format -- all before any device"""
    from occdepth_b200.deploy import _frame_call
    g = _lib.ModelGeom()
    g.V, g.dataset = 2, 0
    nv12 = np.zeros((2, 555, 1242), np.uint8)
    f = {"img": nv12, "cam_k": np.stack([np.eye(3)] * 2), "T_velo_2_cam": np.stack([np.eye(4)] * 2),
         "pixel_format": "nv12"}
    call = lambda fr, fmt: _frame_call(g, fr, None, None, True, None, False, fmt, "who")   # noqa: E731
    with pytest.raises(ValueError, match="pixel_format is 'nv12', this call stages 'rgb'"):
        call(f, "rgb")
    with pytest.raises(ValueError, match="rect_maps"):
        call(dict(f, rect_maps=np.zeros((2, 2, 4, 4), np.float32)), "nv12")
    with pytest.raises(ValueError, match="2 uint8 images"):           # one NV12 image read as two views
        call(dict(f, img=nv12[0]), "nv12")
    with pytest.raises(ValueError, match="2 uint8 images"):           # NV12 bytes staged as RGB
        call(dict(f, pixel_format="rgb"), "rgb")
    with pytest.raises(ValueError, match="2 uint8 images"):           # an odd width
        call(dict(f, img=np.zeros((2, 555, 1241), np.uint8)), "nv12")
    with pytest.raises(ValueError, match="pixel_format must be"):
        deploy.LoadedModel.run_frames(None, [f], pixel_format="yuv")
