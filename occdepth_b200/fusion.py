"""Scene maps: a sequence's per-frame class probabilities fused into one persistent voxel map on the device.

Naive-Bayes semantic mapping keeps, per voxel, a posterior proportional to prod_t p_t(c).  Its log is a sum of
ln p_t(c), and softmax over that sum is the normalised posterior, so the accumulator -- fp32 [C, MX, MY, MZ] -- is a
logits tensor: `classes()` and `voxels()` read it with the class-map kernels and `occupied_voxels` as they are.

    smap = SceneMap(20, (512, 512, 32), 0.2, origin=(-51.2, -51.2, -3.0), device="cuda")
    model.fuse_frames(smap, frames, poses)          # KITTI: poses[i] = world <- velodyne of frame i
    cmap = smap.classes()                           # uint16 [MX, MY, MZ], 255 where no frame looked
    fov_rows, _ = smap.voxels().rows()

`integrate` takes a frame's float16 probabilities over its output grid and the rigid pose of that grid in the map
frame.  Each map voxel centre is taken into the frame grid in float64 (`occd_scene_map_integrate`; the header states
the arithmetic) and, when it lands inside the grid, inside the FOV mask and on no NaN, adds logf(max(p, min_prob)) to
its C accumulators and 1 to its count.  Nearest-voxel lookup, no decay; `shift` moves a streaming map by whole voxels.
Nothing here synchronises with the host.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_CLASSES = 64        # the class-map kernels' LUT cap


def _vec3(v, what, who="SceneMap"):
    a = np.asarray(v, dtype=np.float64).reshape(-1)
    if a.shape != (3,) or not np.isfinite(a).all():
        raise ValueError("%s: %s must hold 3 finite values" % (who, what))
    return a


def check_pose(pose, who="SceneMap.integrate", what="pose"):
    """(T, inverse(T)) in float64 of a finite, invertible 4x4 pose; ValueError otherwise, naming `who` and `what`"""
    if isinstance(pose, torch.Tensor):
        pose = pose.detach().cpu().double().numpy()
    T = np.asarray(pose, dtype=np.float64)
    if T.shape != (4, 4) or not np.isfinite(T).all():
        raise ValueError("%s: %s must be a finite 4x4 matrix" % (who, what))
    try:
        R = np.linalg.inv(T)
    except np.linalg.LinAlgError:
        raise ValueError("%s: %s is singular" % (who, what)) from None
    if not np.isfinite(R).all():
        raise ValueError("%s: %s is singular" % (who, what))
    return T, R


def plane_layout(shape, axes, who="SceneMap.integrate"):
    """(GX, GY, GZ) along the frame grid's x, y, z and their element strides, for one contiguous class plane of
    storage shape (D0, D1, D2): KITTI's output is [x][y][z] ("xyz"), NYU's [x][z][y] ("xzy")"""
    D0, D1, D2 = (int(v) for v in shape)
    if axes == "xyz":
        return (D0, D1, D2), (D1 * D2, D2, 1)
    if axes == "xzy":
        return (D0, D2, D1), (D1 * D2, 1, D2)
    raise ValueError("%s: axes must be 'xyz' or 'xzy', got %r" % (who, axes))


def frame_box(T, grid_origin, grid_voxel, grid_dims, origin, voxel, dims):
    """(i_lo, i_hi, j_lo, j_hi, k_lo, k_hi): the map voxels a frame grid can reach.  The grid's 8 corners taken to the
    map frame by T, their bounding box in map indices, one voxel more on each side, clipped to the map.  A voxel
    centre inside the grid lies inside the corners' hull; the margin covers the rounding of the kernel's float64 path"""
    g = np.asarray(grid_origin, np.float64)
    ext = np.asarray(grid_dims, np.float64) * float(grid_voxel)
    corners = np.array([[g[0] + ext[0] * a, g[1] + ext[1] * b, g[2] + ext[2] * c, 1.0]
                        for a in (0, 1) for b in (0, 1) for c in (0, 1)])
    w = (corners @ np.asarray(T, np.float64).T)[:, :3]
    lo = (w.min(0) - origin) / voxel
    hi = (w.max(0) - origin) / voxel
    box = []
    for a in range(3):
        n = int(dims[a])
        box.append(int(np.clip(np.floor(lo[a]) - 1, 0, n)))
        box.append(int(np.clip(np.floor(hi[a]) + 2, 0, n)))
    return tuple(box)


class SceneMap:
    """An axis-aligned voxel map in a caller-chosen map frame: `origin` (3 float64, the map's corner), `voxel` (edge),
    `dims` (MX, MY, MZ), on one CUDA device.  `acc` fp32 [C, MX, MY, MZ] holds the summed log-probabilities and
    `count` int32 [MX, MY, MZ] the frames that observed each voxel; both start at 0 and are the map's own buffers
    (read them, do not write them).  Frames are integrated in call order; two maps fed the same frames hold the same
    bytes."""

    def __init__(self, n_classes, dims, voxel, origin=(0.0, 0.0, 0.0), device="cuda", min_prob=1e-3):
        n_classes = int(n_classes)
        if not 1 <= n_classes <= MAX_CLASSES:
            raise ValueError("SceneMap: n_classes must be in [1, %d]" % MAX_CLASSES)
        dims = tuple(int(v) for v in dims)
        if len(dims) != 3 or min(dims) < 1:
            raise ValueError("SceneMap: dims must be 3 positive ints")
        voxel = float(voxel)
        if not (np.isfinite(voxel) and voxel > 0):
            raise ValueError("SceneMap: voxel must be finite and positive")
        min_prob = float(min_prob)
        if not 0 < np.float32(min_prob) <= 1:
            raise ValueError("SceneMap: min_prob must be in (0, 1]")
        origin = _vec3(origin, "origin")
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("SceneMap: the map lives on a CUDA device (there is no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.n_classes, self.dims, self.voxel, self.min_prob = n_classes, dims, voxel, min_prob
        self.origin = origin
        self.device = device
        self._acc = torch.zeros((n_classes,) + dims, dtype=torch.float32, device=device)
        self._count = torch.zeros(dims, dtype=torch.int32, device=device)
        self._spare = None      # shift's output pair, allocated at the first shift

    @property
    def acc(self):
        """fp32 [C, MX, MY, MZ]: the summed log-probabilities (a logits tensor)"""
        return self._acc

    @property
    def count(self):
        """int32 [MX, MY, MZ]: how many integrated frames observed each voxel"""
        return self._count

    def reset(self):
        """every voxel back to acc = 0, count = 0 (the geometry stays)"""
        self._acc.zero_()
        self._count.zero_()

    def integrate(self, probs, pose, grid_origin, grid_voxel, axes="xyz", fov_mask=None):
        """Add one frame: probs float16 [C, D0, D1, D2] on the map's device (contiguous; C = the map's classes) over
        a frame grid with corner `grid_origin` and edge `grid_voxel`, stored [x][y][z] (axes="xyz", KITTI) or
        [x][z][y] ("xzy", NYU); pose: the rigid 4x4 taking the frame grid's frame to the map frame.  fov_mask: bool
        or uint8 holding one value per voxel of a class plane, in the same storage order, or None.  Returns the
        launch box (frame_box)."""
        if not isinstance(probs, torch.Tensor) or probs.dtype != torch.float16:
            raise TypeError("SceneMap.integrate: probs must be a float16 tensor")
        if probs.device != self.device:
            raise ValueError("SceneMap.integrate: probs on %s, the map on %s" % (probs.device, self.device))
        if probs.dim() != 4 or probs.numel() == 0 or not probs.is_contiguous():
            raise ValueError("SceneMap.integrate: probs must be a contiguous, non-empty [C, D0, D1, D2] tensor")
        if probs.shape[0] != self.n_classes:
            raise ValueError("SceneMap.integrate: probs holds %d classes, the map %d" % (probs.shape[0],
                                                                                         self.n_classes))
        G, s = plane_layout(probs.shape[1:], axes)
        T, R = check_pose(pose)
        g = _vec3(grid_origin, "grid_origin")
        gv = float(grid_voxel)
        if not (np.isfinite(gv) and gv > 0):
            raise ValueError("SceneMap.integrate: grid_voxel must be finite and positive")
        plane = G[0] * G[1] * G[2]
        mask = None
        if fov_mask is not None:
            mask = fov_mask
            if not isinstance(mask, torch.Tensor) or mask.dtype not in (torch.bool, torch.uint8):
                raise TypeError("SceneMap.integrate: fov_mask must be a bool or uint8 tensor")
            if mask.numel() != plane:
                raise ValueError("SceneMap.integrate: fov_mask holds %d values, a class plane %d" % (mask.numel(),
                                                                                                     plane))
            if mask.device != self.device or not mask.is_contiguous():
                raise ValueError("SceneMap.integrate: fov_mask must be contiguous and on the map's device")
        box = frame_box(T, g, gv, G, self.origin, self.voxel, self.dims)
        Rp = np.ascontiguousarray(R[:3], np.float64)
        strides = np.array((plane,) + s, np.int64)
        o = np.ascontiguousarray(self.origin)
        bx = np.array(box, np.int32)
        with torch.cuda.device(self.device):
            rc = _lib.lib().occd_scene_map_integrate(
                self._acc.data_ptr(), self._count.data_ptr(), self.n_classes, *self.dims, self.voxel,
                o.ctypes.data_as(C.c_void_p), probs.data_ptr(), strides.ctypes.data_as(C.c_void_p),
                None if mask is None else mask.data_ptr(), *G, g.ctypes.data_as(C.c_void_p), gv,
                Rp.ctypes.data_as(C.c_void_p), self.min_prob, bx.ctypes.data_as(C.c_void_p), _lib.stream_ptr())
            _lib.check(rc, "occd_scene_map_integrate")
        return box

    def shift(self, d):
        """Move the map by whole voxels d = (dx, dy, dz): voxel idx afterwards is voxel idx + d before, voxels that
        come into view are unobserved, and origin += d * voxel.  Copies into a second pair of buffers the map owns,
        then swaps them."""
        d = np.asarray(d).reshape(-1)
        if d.shape != (3,) or not all(float(v).is_integer() for v in d):
            raise ValueError("SceneMap.shift: d must hold 3 whole voxel counts")
        d = np.array([int(v) for v in d], np.int32)
        if self._spare is None:
            self._spare = (torch.empty_like(self._acc), torch.empty_like(self._count))
        a2, c2 = self._spare
        with torch.cuda.device(self.device):
            rc = _lib.lib().occd_scene_map_shift(self._acc.data_ptr(), self._count.data_ptr(), a2.data_ptr(),
                                                 c2.data_ptr(), self.n_classes, *self.dims,
                                                 d.ctypes.data_as(C.c_void_p), _lib.stream_ptr())
            _lib.check(rc, "occd_scene_map_shift")
        self._spare = (self._acc, self._count)
        self._acc, self._count = a2, c2
        self.origin = self.origin + d.astype(np.float64) * self.voxel

    def classes(self, inv_map=None, unknown=255, confidence=False, probabilities=False):
        """The fused class map: uint16 [MX, MY, MZ], `OccDepth.class_map` of acc (the same remap, first-max tie rule,
        confidence and probabilities), then `unknown` wherever no frame observed the voxel.  With confidence /
        probabilities: (map, conf [MX, MY, MZ]) / (map, probs [C, MX, MY, MZ]), float16; an unobserved voxel keeps
        what softmax of zeros gives there (1 / C)."""
        from .models.OccDepth import OccDepth
        unknown = int(unknown)
        if not 0 <= unknown <= 65535:
            raise ValueError("SceneMap.classes: unknown must be a uint16 class id")
        with torch.cuda.device(self.device):
            res = OccDepth.class_map(self._acc[None], inv_map, confidence, probabilities)
            cmap = res[0] if isinstance(res, tuple) else res
            rc = _lib.lib().occd_scene_map_mark_unobserved(cmap.data_ptr(), self._count.data_ptr(), cmap.numel(),
                                                           unknown, _lib.stream_ptr())
            _lib.check(rc, "occd_scene_map_mark_unobserved")
        if isinstance(res, tuple):
            return res[0][0], res[1][0]
        return cmap[0]

    def voxels(self, inv_map=None, unknown=255, capacity=None, out=None):
        """`voxels.occupied_voxels` of `classes(inv_map, unknown)` with map-frame centres (the map's voxel and
        origin); `unknown` voxels are skipped as the ignore id"""
        from .voxels import occupied_voxels
        cmap = self.classes(inv_map, unknown)
        with torch.cuda.device(self.device):
            return occupied_voxels(cmap, voxel_size=self.voxel, vox_origin=self.origin, capacity=capacity,
                                   ignore=int(unknown), out=out)

    def render(self, E, K, size, inv_map=None, unknown=255, near=0.0, far=float("inf")):
        """The map as a camera sees it: `render.render_classes` of `classes(inv_map, unknown)` with the map's origin
        and voxel ("xyz").  E: the 4x4 map frame -> camera frame (or (1, V, 4, 4) for V cameras), K the 3x3
        intrinsics, size = (W, H).  Unobserved voxels are transparent (ignore = unknown); class 0 is empty.
        Returns View(classes, depth, index), each [1, V, H, W]."""
        from .render import check_request, render_classes
        unknown = int(unknown)
        if not 0 <= unknown <= 65535:
            raise ValueError("SceneMap.render: unknown must be a uint16 class id")
        args = dict(E=E, K=K, size=size, grid_origin=self.origin, grid_voxel=self.voxel, ignore=unknown, near=near,
                    far=far, who="SceneMap.render")
        check_request(1, self.dims, **args)           # every refusal before classes() launches
        cmap = self.classes(inv_map, unknown)
        with torch.cuda.device(self.device):
            return render_classes(cmap, **args)

    def render_probs(self, E, K, size, inv_map=None, unknown=255, near=0.0, far=float("inf"),
                     min_transmittance=1e-4):
        """The fused posterior as a camera sees it: `render.render_probs` of `classes(inv_map, unknown,
        probabilities=True)`, with that map as class_map and ignore = unknown, so unobserved voxels are transparent
        (rather than opaque at 1 / C per class); class 0 is empty.  inv_map remaps the returned classes only.
        Returns SoftView(classes, depth, opacity, probs), each [1, V, ...]."""
        from .render import check_request, render_probs
        unknown = int(unknown)
        if not 0 <= unknown <= 65535:
            raise ValueError("SceneMap.render_probs: unknown must be a uint16 class id")
        t_min = float(np.float32(min_transmittance))
        if not 0.0 <= t_min < 1.0:
            raise ValueError("SceneMap.render_probs: min_transmittance must be in [0, 1), got %r" % (min_transmittance,))
        lut = None
        if inv_map is not None:
            lut = np.asarray(inv_map).reshape(-1)
            if lut.shape != (self.n_classes,):
                raise ValueError("SceneMap.render_probs: inv_map must hold one label id per class (%d)"
                                 % self.n_classes)
        args = dict(E=E, K=K, size=size, grid_origin=self.origin, grid_voxel=self.voxel, ignore=unknown, near=near,
                    far=far, who="SceneMap.render_probs")
        check_request(1, self.dims, **args, n_classes=self.n_classes)    # every refusal before classes() launches
        cmap, probs = self.classes(inv_map, unknown, probabilities=True)
        with torch.cuda.device(self.device):
            return render_probs(probs, **args, class_map=cmap, min_transmittance=t_min, inv_map=lut)
