"""Camera views of a class map: for each pixel, the first occupied voxel along its ray, with its class, depth and
voxel index, computed on the device; and soft views of class probabilities (render_probs): each ray composited
through every voxel's float16 probabilities into an expected depth, an opacity and a per-pixel class distribution.

    view = render_classes(cmap, E, K, (1220, 370), vox_origin, 0.2)   # cmap uint16 [B, 256, 256, 32] ([x][y][z])
    view.classes    # uint16 [B, V, H, W]: the hit voxel's class, `empty` where the ray meets nothing
    view.depth      # float32: the camera-frame z at which the ray enters that voxel, +inf on a miss
    view.index      # int32: the voxel's flat index in its map (what occupied_voxels rows carry), -1 on a miss

This is what a user overlays on the image, or compares with a depth map, to check a semantic occupancy prediction
against the camera: the prediction as that camera sees it.  `occd_render_classes` walks each ray voxel by voxel
(Amanatides-Woo) in float64 with explicit rounding; include/occdepth_b200.h states the arithmetic.  The host builds
each camera's 12 float64 values from E and K; nothing here synchronises with the host or copies to the device.
"""
import ctypes as C
from collections import namedtuple

import numpy as np
import torch

from . import _lib
from .fusion import _vec3, check_pose, plane_layout

MAX_CAMERAS = 32        # OCCD_RENDER_MAX_CAMERAS: the cameras of one call travel in the kernel parameters

View = namedtuple("View", ["classes", "depth", "index"])
View.__doc__ = """one call's outputs, each [B, V, H, W] or None: classes uint16, depth float32, index int32"""

SoftView = namedtuple("SoftView", ["classes", "depth", "opacity", "probs"])
SoftView.__doc__ = """one soft render's outputs or None: classes uint16, depth and opacity float32 [B, V, H, W], probs
float16 [B, V, C, H, W]"""

_DTYPES = (torch.uint16, torch.float32, torch.int32)
_SOFT_DTYPES = (torch.uint16, torch.float32, torch.float32, torch.float16)


def _lead(a, B, what, who):
    """a (4, 4) / (3, 3) matrix, (B, ...) or (B, V, ...) as float64 (B, V', ...)"""
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().double().numpy()
    a = np.asarray(a, dtype=np.float64)
    n = 4 if what == "E" else 3
    if a.ndim < 2 or a.shape[-2:] != (n, n) or a.ndim > 4:
        raise ValueError("%s: %s must be (%d, %d), (B, %d, %d) or (B, V, %d, %d), got %r"
                         % (who, what, n, n, n, n, n, n, a.shape))
    if a.ndim == 2:
        a = np.broadcast_to(a, (B, 1, n, n))
    elif a.ndim == 3:
        a = a[:, None]
    if a.shape[0] != B:
        raise ValueError("%s: %s holds %d items, the class map %d" % (who, what, a.shape[0], B))
    return a


def _camera(E, K, who):
    """the 12 float64 values of one camera: M = R^-1 K^-1 (row-major) and o = -R^-1 t, from inverse(E)"""
    _, Ei = check_pose(E, who, "E")
    if not np.isfinite(K).all():
        raise ValueError("%s: K must be finite" % who)
    if tuple(K[2]) != (0.0, 0.0, 1.0):
        raise ValueError("%s: K's last row must be (0, 0, 1), got %r" % (who, tuple(K[2])))
    try:
        Ki = np.linalg.inv(K)
    except np.linalg.LinAlgError:
        raise ValueError("%s: K is singular" % who) from None
    M = Ei[:3, :3] @ Ki
    if not np.isfinite(M).all():
        raise ValueError("%s: K is singular" % who)
    return np.concatenate([M.reshape(-1), Ei[:3, 3]])


def cameras(E, K, B=1, who="render_classes"):
    """float64 (B, V, 12): every camera of a call, E and K broadcast against each other over (B, V)"""
    E = _lead(E, B, "E", who)
    K = _lead(K, B, "K", who)
    V = max(E.shape[1], K.shape[1])
    if E.shape[1] not in (1, V) or K.shape[1] not in (1, V):
        raise ValueError("%s: E holds %d cameras per item, K %d" % (who, E.shape[1], K.shape[1]))
    if B * V > MAX_CAMERAS:
        raise ValueError("%s: %d maps x %d cameras, at most %d cameras per call" % (who, B, V, MAX_CAMERAS))
    out = np.empty((B, V, 12), np.float64)
    for b in range(B):
        for v in range(V):
            out[b, v] = _camera(E[b, v if E.shape[1] > 1 else 0], K[b, v if K.shape[1] > 1 else 0], who)
    return out


def check_request(B, storage, E, K, size, grid_origin, grid_voxel, axes="xyz", empty=0, ignore=255, near=0.0,
                  far=float("inf"), who="render_classes", n_classes=None):
    """Every host-side check of a render of B maps of storage shape `storage` (D0, D1, D2): the launch's arguments
    (G, s, W, H, origin, voxel, empty, ignore, near, far, cams), or ValueError naming `who`.  n_classes: a soft
    render's channel count, below which `empty` (a channel index there) must lie"""
    G, s = plane_layout(storage, axes, who)
    if G[0] * G[1] * G[2] > 2 ** 31 - 1:
        raise ValueError("%s: a map holds at most 2^31 - 1 voxels" % who)
    try:
        W, H = (int(x) for x in size)
    except (TypeError, ValueError):
        raise ValueError("%s: size must be (W, H)" % who) from None
    if W <= 0 or H <= 0 or H > 65535 or W * H > 2 ** 31 - 1:
        raise ValueError("%s: size (W, H) must be positive, H <= 65535 and W * H < 2^31, got %r" % (who, (W, H)))
    origin = _vec3(grid_origin, "grid_origin", who)
    voxel = float(grid_voxel)
    if not (np.isfinite(voxel) and voxel > 0):
        raise ValueError("%s: grid_voxel must be finite and positive" % who)
    empty, ignore = int(empty), int(ignore)
    if not (0 <= empty <= 65535 and 0 <= ignore <= 65535):
        raise ValueError("%s: empty and ignore must be uint16 class ids" % who)
    if n_classes is not None and not empty < n_classes:
        raise ValueError("%s: empty (%d) must be a channel index below C = %d" % (who, empty, n_classes))
    near, far = float(near), float(far)
    if not (np.isfinite(near) and near >= 0 and far > near):
        raise ValueError("%s: near must be finite and >= 0, far > near (got %r, %r)" % (who, near, far))
    cams = cameras(E, K, B, who)
    return dict(G=G, s=s, W=W, H=H, origin=origin, voxel=voxel, empty=empty, ignore=ignore, near=near, far=far,
                cams=cams)


def _outputs(out, fields, dtypes, shapes, device, who):
    """`out` checked against the expected dtypes and shapes (None entries are not computed), or freshly allocated"""
    if out is None:
        return tuple(torch.empty(sh, dtype=dt, device=device) for dt, sh in zip(dtypes, shapes))
    out = tuple(out)
    if all(x is None for x in out):
        raise ValueError("%s: out must hold at least one output" % who)
    for name, x, dt, shape in zip(fields, out, dtypes, shapes):
        if x is None:
            continue
        if not isinstance(x, torch.Tensor) or x.dtype != dt:
            raise TypeError("%s: out.%s must be a %s tensor" % (who, name, dt))
        if tuple(x.shape) != shape or x.device != device or not x.is_contiguous():
            raise ValueError("%s: out.%s must be contiguous %r on %s" % (who, name, shape, device))
    return out


def render_classes(class_map, E, K, size, grid_origin, grid_voxel, axes="xyz", empty=0, ignore=255, near=0.0,
                   far=float("inf"), out=None, who="render_classes"):
    """Cast one ray per pixel through `class_map` and return View(classes, depth, index), each [B, V, H, W].

    class_map: uint16 [B, D0, D1, D2] or [D0, D1, D2] (then B = 1), contiguous, on a CUDA device, stored [x][y][z]
      (axes="xyz", KITTI's output) or [x][z][y] ("xzy", NYU's); the grid has corner `grid_origin` (3 values) and
      edge `grid_voxel`.
    E: the 4x4 taking the grid's frame to the camera frame (KITTI T_velo_2_cam, NYU world -> cam), K: the 3x3
      intrinsics with last row (0, 0, 1); each (.., ..), (B, ..) or (B, V, ..), broadcast against each other.  At most
      32 cameras (B x V) per call.  size = (W, H); pixel (u, v) is the image point (u, v).
    A voxel stops the ray when its class is neither `empty` nor `ignore`; only the part of the ray with camera z in
    [near, far] counts.  depth is that camera z where the ray enters the hit voxel (+inf on a miss); index is the
    voxel's flat index in its map (-1 on a miss); classes holds `empty` on a miss.
    out: a View of preallocated outputs; an entry that is None is not computed (at least one must be given).
    Everything is checked on the host before the launch; one launch on the current stream.  `who` names the caller
    in the refusals."""
    if not isinstance(class_map, torch.Tensor) or class_map.dtype != torch.uint16:
        raise TypeError("%s: class_map must be a uint16 tensor" % who)
    if class_map.dim() == 3:
        class_map = class_map.unsqueeze(0)
    if class_map.dim() != 4 or class_map.numel() == 0 or not class_map.is_contiguous():
        raise ValueError("%s: class_map must be a contiguous, non-empty [B, D0, D1, D2] or [D0, D1, D2] tensor" % who)
    B = int(class_map.shape[0])
    a = check_request(B, class_map.shape[1:], E, K, size, grid_origin, grid_voxel, axes, empty, ignore, near, far,
                      who)
    V = a["cams"].shape[1]
    shape = (B, V, a["H"], a["W"])
    out = View(*_outputs(out, View._fields, _DTYPES, (shape,) * 3, class_map.device, who))
    if class_map.device.type != "cuda":
        raise ValueError("%s: class_map must be on a CUDA device (there is no CPU fallback)" % who)
    st = np.array(a["s"], np.int64)
    cam = np.ascontiguousarray(a["cams"])
    ptr = lambda x: None if x is None else x.data_ptr()      # noqa: E731
    with torch.cuda.device(class_map.device):
        rc = _lib.lib().occd_render_classes(class_map.data_ptr(), B, *a["G"], st.ctypes.data_as(C.c_void_p),
                                            a["origin"].ctypes.data_as(C.c_void_p), a["voxel"], V,
                                            cam.ctypes.data_as(C.c_void_p), a["W"], a["H"], a["empty"], a["ignore"],
                                            a["near"], a["far"], ptr(out.classes), ptr(out.depth), ptr(out.index),
                                            _lib.stream_ptr())
        _lib.check(rc, "occd_render_classes")
    return out


def render_probs(probs, E, K, size, grid_origin, grid_voxel, axes="xyz", class_map=None, empty=0, ignore=255,
                 near=0.0, far=float("inf"), min_transmittance=1e-4, inv_map=None, out=None, who="render_probs"):
    """Composite each pixel's ray front to back through per-voxel class probabilities and return SoftView(classes,
    depth, opacity, probs).

    probs: float16 [B, C, D0, D1, D2] or [C, D0, D1, D2] (then B = 1), contiguous, on a CUDA device -- what
      predict_frame(s)(probabilities=True) or SceneMap.classes(probabilities=True) return -- stored as `axes` says
      (render_classes); 1 <= C <= 64, channel `empty` the chance a voxel is free.  E, K, size, grid_origin,
      grid_voxel, near and far as in render_classes.
    class_map: optional uint16 [B, D0, D1, D2] (or [D0, D1, D2]) of the same grid; voxels holding `ignore` there are
      skipped (transparent).
    Walking the voxels render_classes walks, each voxel is occupied with probability 1 - p(empty), independently, and
    then has class c with weight p(c): T (the chance the ray is still unblocked) falls by p(empty) per voxel, voxel i
    adds T p_i(c) to channel c, in float32 as include/occdepth_b200.h states; the walk stops once T <=
    min_transmittance (in [0, 1); 0 walks every voxel).  Per pixel: opacity = 1 - T, depth = the expected entry depth
    of the first occupied voxel (+inf where opacity is 0), probs [B, V, C, H, W] the channels (channel `empty` is T:
    the ray leaves unblocked), classes the first largest channel, remapped through inv_map (C label ids) when given.
    out: a SoftView of preallocated outputs; an entry that is None is not computed (at least one must be given).
    Everything is checked on the host before the launch; one launch on the current stream."""
    if not isinstance(probs, torch.Tensor) or probs.dtype != torch.float16:
        raise TypeError("%s: probs must be a float16 tensor" % who)
    if probs.dim() == 4:
        probs = probs.unsqueeze(0)
    if probs.dim() != 5 or probs.numel() == 0 or not probs.is_contiguous():
        raise ValueError("%s: probs must be a contiguous, non-empty [B, C, D0, D1, D2] or [C, D0, D1, D2] tensor"
                         % who)
    B, Cn = int(probs.shape[0]), int(probs.shape[1])
    if Cn > 64:
        raise ValueError("%s: probs holds %d classes, at most 64" % (who, Cn))
    storage = tuple(probs.shape[2:])
    if class_map is not None:
        if not isinstance(class_map, torch.Tensor) or class_map.dtype != torch.uint16:
            raise TypeError("%s: class_map must be a uint16 tensor" % who)
        if class_map.dim() == 3:
            class_map = class_map.unsqueeze(0)
        if tuple(class_map.shape) != (B,) + storage or not class_map.is_contiguous():
            raise ValueError("%s: class_map must be contiguous %r, the probabilities' grid"
                             % (who, (B,) + storage))
        if class_map.device != probs.device:
            raise ValueError("%s: class_map and probs must be on the same device" % who)
    a = check_request(B, storage, E, K, size, grid_origin, grid_voxel, axes, empty, ignore, near, far, who, Cn)
    t_min = float(np.float32(min_transmittance))          # the kernel's float32 threshold
    if not 0.0 <= t_min < 1.0:
        raise ValueError("%s: min_transmittance must be in [0, 1), got %r" % (who, min_transmittance))
    lut = None
    if inv_map is not None:
        lut = np.ascontiguousarray(np.asarray(inv_map).astype(np.int32))
        if lut.shape != (Cn,):
            raise ValueError("%s: inv_map must hold one label id per class (%d)" % (who, Cn))
    V = a["cams"].shape[1]
    shape = (B, V, a["H"], a["W"])
    out = SoftView(*_outputs(out, SoftView._fields, _SOFT_DTYPES, (shape,) * 3 + ((B, V, Cn, a["H"], a["W"]),),
                             probs.device, who))
    if probs.device.type != "cuda":
        raise ValueError("%s: probs must be on a CUDA device (there is no CPU fallback)" % who)
    st = np.array(a["s"], np.int64)
    cam = np.ascontiguousarray(a["cams"])
    ptr = lambda x: None if x is None else x.data_ptr()      # noqa: E731
    with torch.cuda.device(probs.device):
        rc = _lib.lib().occd_render_probs(probs.data_ptr(), B, Cn, *a["G"], st.ctypes.data_as(C.c_void_p),
                                          ptr(class_map), a["ignore"], a["empty"],
                                          a["origin"].ctypes.data_as(C.c_void_p), a["voxel"], V,
                                          cam.ctypes.data_as(C.c_void_p), a["W"], a["H"], a["near"], a["far"], t_min,
                                          None if lut is None else lut.ctypes.data_as(C.c_void_p), ptr(out.classes),
                                          ptr(out.depth), ptr(out.opacity), ptr(out.probs), _lib.stream_ptr())
        _lib.check(rc, "occd_render_probs")
    return out
