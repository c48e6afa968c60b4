"""ctypes binding of include/occdepth_b200.h (the C-ABI drop-in boundary).

The library is mandatory: there is no CPU or PyTorch fallback behind these calls.  `lib()` raises if
libocc_b200.so has not been built (python -m occdepth_b200._build / __graft_entry__.build()).
"""
import ctypes as C
import os
import threading

from . import _build

_LIB = None

MAX_SCALES = 4
DTYPE_F32, DTYPE_BF16 = 0, 1
DTYPE_U8, DTYPE_U16, DTYPE_I64 = 2, 3, 4
PIX_RGB, PIX_BGR, PIX_NV12 = 0, 1, 2
PIXEL_FORMATS = {"rgb": PIX_RGB, "bgr": PIX_BGR, "nv12": PIX_NV12}
SFA_OUT_F32_PLANAR, SFA_OUT_BF16_CL, SFA_OUT_F32_CL, SFA_OUT_TF32_CL = 0, 1, 2, 3
ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_SILU, ACT_SIGMOID = 0, 1, 2, 3, 4


class SfaParams(C.Structure):
    _fields_ = [
        ("feat", C.c_void_p * MAX_SCALES),
        ("h", C.c_int * MAX_SCALES),
        ("w", C.c_int * MAX_SCALES),
        ("div", C.c_int * MAX_SCALES),
        ("vstride", C.c_longlong * MAX_SCALES),
        ("n_scales", C.c_int),
        ("n_views", C.c_int),
        ("C", C.c_int),
        ("feat_dtype", C.c_int),
        ("pix", C.c_void_p),
        ("fov", C.c_void_p),
        ("N", C.c_longlong),
        ("P", C.c_int),
        ("out", C.c_void_p),
        ("out_mode", C.c_int),
        ("out_cstride", C.c_int),
        ("perm_nyu", C.c_int),
        ("S1", C.c_int),
        ("S2", C.c_int),
        ("prior", C.c_void_p),
        ("scale_const", C.c_float),
    ]


CONV_MAX_TAPS, CONV_MAX_SRC, CONV_MAX_GROUPS = 81, 3, 8
CONV_IMPL_TC, CONV_IMPL_SIMT, CONV_IMPL_HALO, CONV_IMPL_HALOX, CONV_IMPL_TCX, CONV_IMPL_AUTO = 0, 1, 2, 3, 4, 5
OUT1_NONE, OUT1_CL, OUT1_F32_PLANAR, OUT1_CLASS_U16, OUT1_CLASS_U16_CONF, OUT1_CLASS_U16_PROBS = 0, 1, 2, 3, 4, 5
CLASS_LUT_MAX = 64
ERR_ARG, ERR_CUDA, ERR_UNSUPPORTED, ERR_FORMAT, ERR_IO = 1, 2, 3, 4, 5
MODEL_FORMAT_VERSION = 1
FRAME_NO_GRAPH = 1


class ModelGeom(C.Structure):
    """occd_model_geom"""
    _fields_ = [("precision", C.c_int), ("dataset", C.c_int), ("V", C.c_int), ("img_h", C.c_int),
                ("img_w", C.c_int), ("project_scale", C.c_int), ("X", C.c_int), ("Y", C.c_int), ("Z", C.c_int),
                ("n_classes", C.c_int), ("has_depth", C.c_int), ("depth_h", C.c_int), ("depth_w", C.c_int),
                ("flosp_depth", C.c_int), ("graph", C.c_int), ("device_bytes", C.c_longlong),
                ("voxel_size", C.c_double), ("vox_origin", C.c_double * 3), ("scene_size", C.c_double * 3)]


class Frame(C.Structure):
    """occd_frame"""
    _fields_ = [("images", C.c_void_p), ("img_stride", C.c_longlong), ("row_stride", C.c_longlong),
                ("H0", C.c_int), ("W0", C.c_int), ("cam_k", C.c_void_p), ("pose", C.c_void_p),
                ("calib_f32", C.c_int), ("vox_origin", C.c_void_p), ("scene_size", C.c_void_p),
                ("voxel_size", C.c_double), ("depth", C.c_void_p), ("depth_h", C.c_int), ("depth_w", C.c_int),
                ("flags", C.c_int)]


class FrameEx(C.Structure):
    """occd_frame_ex"""
    _fields_ = [("frame", Frame), ("pixel_format", C.c_int), ("uv_offset", C.c_longlong)]


class VoxelOut(C.Structure):
    """occd_voxel_out"""
    _fields_ = [("capacity", C.c_int), ("voxel_size", C.c_double), ("origin", C.c_void_p), ("count", C.c_void_p),
                ("hist", C.c_void_p), ("index", C.c_void_p), ("cls", C.c_void_p), ("xyz", C.c_void_p)]


class ConvTap(C.Structure):
    _fields_ = [("src", C.c_int), ("dz", C.c_int), ("dy", C.c_int), ("dx", C.c_int)]


class ConvDesc(C.Structure):
    _fields_ = [
        ("impl", C.c_int),
        ("dtype", C.c_int),
        ("n_src", C.c_int),
        ("src", C.c_void_p * CONV_MAX_SRC),
        ("src_C", C.c_int * CONV_MAX_SRC),
        ("src_cstride", C.c_int * CONV_MAX_SRC),
        ("src_coff", C.c_int * CONV_MAX_SRC),
        ("B", C.c_int), ("ID", C.c_int), ("IH", C.c_int), ("IW", C.c_int),
        ("src_d0", C.c_int),
        ("stride", C.c_int * 3),
        ("n_taps", C.c_int),
        ("taps", ConvTap * CONV_MAX_TAPS),
        ("weight", C.c_void_p),
        ("bias", C.c_void_p),
        ("Cout", C.c_int), ("Cout_pad", C.c_int), ("Kpad", C.c_int),
        ("weight_per_image", C.c_int),
        ("OD", C.c_int), ("OH", C.c_int), ("OW", C.c_int),
        ("omul", C.c_int * 3), ("oadd", C.c_int * 3),
        ("ODf", C.c_int), ("OHf", C.c_int), ("OWf", C.c_int),
        ("out0", C.c_void_p),
        ("out0_cstride", C.c_int), ("out0_coff", C.c_int),
        ("act", C.c_int),
        ("out0_exact", C.c_int),
        ("res1", C.c_void_p),
        ("res1_cstride", C.c_int), ("res1_coff", C.c_int),
        ("res2", C.c_void_p),
        ("res2_cstride", C.c_int), ("res2_coff", C.c_int),
        ("res2_post", C.c_int),
        ("out1_mode", C.c_int),
        ("out1", C.c_void_p),
        ("out1_cstride", C.c_int), ("out1_coff", C.c_int),
        ("out1_C", C.c_int),
        ("n_groups", C.c_int),
        ("group_tap0", C.c_int * (CONV_MAX_GROUPS + 1)),
        ("group_oadd", (C.c_int * 3) * CONV_MAX_GROUPS),
    ]


# every symbol include/occdepth_b200.h declares: name -> (restype, argtypes)
_vp, _i, _ll, _f = C.c_void_p, C.c_int, C.c_longlong, C.c_float
SYMBOLS = {
    "occd_abi_version": (C.c_int, []),
    "occd_last_error": (C.c_char_p, []),
    "occd_sfa_lift_fwd": (C.c_int, [C.POINTER(SfaParams), _vp]),
    "occd_planar_to_cl": (C.c_int, [_vp, _vp, _i, _ll, _i, _ll, _i, _vp]),
    "occd_cl_to_planar": (C.c_int, [_vp, _i, _vp, _ll, _i, _ll, _i, _vp]),
    "occd_conv_plan_create": (C.c_int, [C.POINTER(ConvDesc), C.POINTER(C.c_void_p)]),
    "occd_conv_plan_destroy": (C.c_int, [_vp]),
    "occd_conv_run": (C.c_int, [_vp, _vp]),
    "occd_conv_plan_info": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "occd_conv_plan_impl": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "occd_conv_plan_schedule": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "occd_conv_plan_set_class_lut": (C.c_int, [_vp, _vp, _i]),
    "occd_conv_debug_trace": (C.c_int, [_vp]),
    "occd_softmax_planar_to_cl": (C.c_int, [_vp, _vp, _i, _ll, _i, _ll, _i, _i, _vp]),
    "occd_argmax_classes": (C.c_int, [_vp, _vp, _ll, _i, _ll, _vp, _vp]),
    "occd_argmax_classes_conf": (C.c_int, [_vp, _vp, _vp, _ll, _i, _ll, _vp, _vp]),
    "occd_class_probs": (C.c_int, [_vp, _vp, _vp, _ll, _i, _ll, _vp, _vp]),
    "occd_normalize_rgb_u8": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "occd_stage_rgb_u8_cl": (C.c_int, [_vp, _ll, _ll, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp]),
    "occd_stage_camera_u8_cl": (C.c_int, [_vp, _i, _ll, _ll, _ll, _i, _i, _i, _i, _i, _vp, _ll, _vp, _vp, _vp, _i,
                                          _i, _vp]),
    "occd_depth_u16_to_f32": (C.c_int, [_vp, _vp, _ll, C.c_double, _f, _vp]),
    "occd_vox2pix_fwd": (C.c_int, [_vp, _i, _vp, _vp, C.c_double, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp]),
    "occd_vox2pix_range_fwd": (C.c_int, [_vp, _i, _vp, _vp, C.c_double, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp,
                                         _ll, _ll, _vp]),
    "occd_cl_transpose": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _ll, _vp]),
    "occd_copy_channels": (C.c_int, [_vp, _vp, _i, _ll, _i, _i, _i, _i, _i, _vp]),
    "occd_dwconv2d_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp] + [_i] * 14 + [_vp]),
    "occd_dwconv2d_tiled_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _vp] + [_i] * 14 + [_vp]),
    "occd_se_gate_fwd": (C.c_int, [_vp, _f, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "occd_se_gate_fold_fwd": (C.c_int, [_vp, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "occd_scale_weights": (C.c_int, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "occd_frustum_sample_fwd": (C.c_int, [_vp, _vp] + [_i] * 7 + [_f] * 4 + [_i, _vp, _i, _vp]),
    "occd_grid_sample_prior_fwd": (C.c_int, [_vp, _vp] + [_i] * 8 + [_vp, _i, _vp]),
    "occd_frustum_sample_window_fwd": (C.c_int, [_vp, _vp] + [_i] * 9 + [_f] * 4 + [_i, _vp, _i, _vp]),
    "occd_grid_sample_prior_window_fwd": (C.c_int, [_vp, _vp] + [_i] * 10 + [_vp, _i, _vp]),
    "occd_softmax_planar": (C.c_int, [_vp, _vp, _ll, _i, _ll, _vp]),
    "occd_fc_fwd": (C.c_int, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "occd_channel_scale": (C.c_int, [_vp, _vp, _i, _ll, _ll, _i, _i, _vp]),
    "occd_virtual_view_fwd": (C.c_int, [_vp, _vp, _vp] + [_i] * 9 + [_f, _vp]),
    "occd_virtual_view_items_fwd": (C.c_int, [_vp, _vp, _vp] + [_i] * 9 + [_f, _ll, _vp]),
    "occd_upsample_bilinear_ac": (C.c_int, [_vp, _vp] + [_i] * 11 + [_vp]),
    "occd_upsample_tapsum_ac": (C.c_int, [_vp, _vp, _vp] + [_i] * 15 + [_vp]),
    "occd_ssc_confusion": (C.c_int, [_vp, _i, _vp, _i, _ll, _i, _vp, _vp]),
    "occd_ssc_loss_sums": (C.c_int, [_vp, _vp, _i, _i, _i, _ll, _vp, _vp, _vp, _vp, _i, _vp, _vp, _ll, _vp]),
    "occd_crp_relation_sums": (C.c_int, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _ll, _vp]),
    "occd_depth_cls_sums": (C.c_int, [_vp, _i, _i, _i, _vp, _i, _i, _i, _i, C.c_double, C.c_double, _vp, _vp, _ll,
                                      _vp]),
    "occd_occupied_voxels": (C.c_int, [_vp, _vp] + [_i] * 9 + [_vp] * 5 + [C.c_double, _vp, _vp, _ll, _vp]),
    "occd_model_load": (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    "occd_model_info": (C.c_int, [_vp, C.POINTER(ModelGeom)]),
    "occd_model_run_frame": (C.c_int, [_vp, C.POINTER(Frame), _vp, _vp]),
    "occd_model_run_frame_conf": (C.c_int, [_vp, C.POINTER(Frame), _vp, _vp, _vp]),
    "occd_model_batch": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "occd_model_run_frames": (C.c_int, [_vp, C.POINTER(Frame), _i, _vp, _vp, _vp]),
    "occd_model_run_frames_ex": (C.c_int, [_vp, C.POINTER(FrameEx), _i, _vp, _vp, _vp]),
    "occd_model_list_voxels": (C.c_int, [_vp, _i, C.POINTER(VoxelOut), _vp]),
    "occd_model_run_frames_probs": (C.c_int, [_vp, C.POINTER(FrameEx), _i, _vp, _vp, _vp]),
    "occd_model_destroy": (C.c_int, [_vp]),
    "occd_flosp_camera_tables": (C.c_int, [_i, _vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "occd_comm_halo_exchange": (C.c_int, [_vp, _vp, _ll, _i, _i, _vp]),
    "occd_comm_all_gather": (C.c_int, [_vp, _vp, _vp, _ll, _vp]),
    "occd_comm_gather_root": (C.c_int, [_vp, _vp, _vp, _vp, _ll, _vp]),
    "occd_comm_gather_root_items": (C.c_int, [_vp, _vp, _vp, _vp, _ll, _i, _vp]),
}
# include/occdepth_b200_comm.h: communicators and slab model files; none of these is a launch a model file records
COMM_SYMBOLS = {
    "occd_comm_unique_id": (C.c_int, [C.c_char_p, _vp]),
    "occd_comm_create": (C.c_int, [C.c_char_p, _vp, _i, _i, C.POINTER(C.c_void_p)]),
    "occd_comm_create_local": (C.c_int, [_i, C.POINTER(C.c_void_p)]),
    "occd_comm_destroy": (C.c_int, [_vp]),
    "occd_model_load_slab": (C.c_int, [C.c_char_p, _vp, C.POINTER(C.c_void_p)]),
    "occd_model_run_frame_group": (C.c_int, [C.POINTER(C.c_void_p), _i, C.POINTER(Frame), _vp, _vp, _vp]),
    "occd_model_run_frame_group_probs": (C.c_int, [C.POINTER(C.c_void_p), _i, C.POINTER(Frame), _vp, _vp, _vp]),
}
COMM_ID_BYTES = 128
VOXEL_TILE = 2048


def voxel_work_len(B, N):
    """uint32 elements of occd_occupied_voxels' workspace (OCCD_VOXEL_WORK_LEN)"""
    return 2 * B * ((N + VOXEL_TILE - 1) // VOXEL_TILE)


LOSS_WORK_BLOCKS = 264
SSC_LOSS_MAX_CLASSES = SSC_LOSS_MAX_FRUSTUMS = 64
CRP_MAX_RELATIONS = 16
DEPTH_MAX_BINS = 1024


def ssc_loss_sums_len(C, F):
    """length of occd_ssc_loss_sums' sums for C classes and F frustums (OCCD_SSC_LOSS_SUMS)"""
    return 6 + 3 * C + F * C


# deploy.export: while its thread has `recorder` set, lib() returns that stand-in there (which records the calls it
# forwards); other threads keep the library
_RECORDING = threading.local()
# the communicator argument of a recorded collective: the model file's communicator slot, which the loader fills
MODEL_COMM = object()


def recording():
    """True while deploy.export records a plan's run on this thread: the collective ops then emit the library's
    collective launches (on MODEL_COMM) instead of running"""
    rec = getattr(_RECORDING, "recorder", None)
    return rec is not None and rec.recording


def lib():
    """Load libocc_b200.so (once).  Fails loudly when it is missing -- never falls back."""
    global _LIB
    rec = getattr(_RECORDING, "recorder", None)
    if rec is not None:
        return rec
    if _LIB is None:
        path = _build.lib_path()
        if not os.path.exists(path):
            raise RuntimeError(
                "occdepth_b200: %s is missing -- build it with `python -m occdepth_b200._build` "
                "(or __graft_entry__.build()); there is no CPU fallback" % path)
        L = C.CDLL(path)
        for name, (res, args) in list(SYMBOLS.items()) + list(COMM_SYMBOLS.items()):
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc, what):
    if rc != 0:
        msg = lib().occd_last_error()
        raise RuntimeError("%s failed (code %d): %s" % (what, rc, (msg or b"").decode()))


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
