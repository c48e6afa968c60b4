"""Device-side pieces of the reference's data pipeline (`occdepth.data`), SURVEY 8f row 2.

`vox2pix` mirrors `occdepth.data.utils.helpers.vox2pix` (helpers.py:94-169): same arguments, same three results
(`projected_pix` int64 (N, P, 2), `fov_mask` bool (N, P), `pix_z` (N,) in the pose's precision), bit for bit -- but computed by
`occd_vox2pix_fwd` on the GPU and returned as CUDA tensors, so the 8.4 MB of indices per stereo frame never
cross PCIe and the per-sample numba job disappears from the loader.
"""
import ctypes as C

import numpy as np
import torch

from .. import _lib

# fusion.py:238-330 `pixel_partern` ("dso residual pattern"): (dx, dy) offsets around the projected centre
PIXEL_PATTERNS = [
    [[0, 0]],
    [[0, 0], [0, -1], [-1, 0], [1, 0], [0, 1]],
    [[0, 0], [-1, -1], [1, 1], [-1, 1], [1, -1]],
    [[0, 0], [-1, -1], [-1, 0], [-1, 1], [-1, 0], [0, 1], [1, -1], [1, 0], [1, 1]],
    [[0, 0], [0, -2], [-1, -1], [1, -1], [-2, 0], [2, 0], [-1, 1], [1, 1], [0, 2]],
    [[0, 0], [0, -2], [-1, -1], [1, -1], [-2, 0], [2, 0], [-1, 1], [1, 1], [0, 2], [-2, -2], [-2, 2], [2, -2],
     [2, 2]],
    [[0, 0]] + [[a, b] for a in (-2, -1, 0, 1, 2) for b in (-2, -1, 0, 1, 2) if (a, b) != (0, 0)],
    [[0, 0], [0, -2], [-1, -1], [1, -1], [-2, 0], [2, 0], [-1, 1], [0, 2]],
    [[0, 0], [0, -2], [-1, -1], [1, -1], [-2, 0], [2, 0], [-1, 1], [1, 1], [0, 2], [-2, -2], [-2, 2], [2, -2],
     [2, 2], [-3, -1], [-3, 1], [3, -1], [3, 1], [1, -3], [-1, -3], [1, 3], [-1, 3]],
]


def volume_dims(vox_origin, voxel_size, scene_size):
    """helpers.py:126-134, the same numpy expression (so the same rounding of the extent)"""
    vol_bnds = np.zeros((3, 2))
    vol_bnds[:, 0] = vox_origin
    vol_bnds[:, 1] = np.asarray(vox_origin) + np.array(scene_size)
    return np.ceil((vol_bnds[:, 1] - vol_bnds[:, 0]) / voxel_size).copy(order="C").astype(int)


def _require_cuda(dev, what):
    if dev.type != "cuda" or not torch.cuda.is_available():
        raise RuntimeError("occdepth_b200.data.%s runs on CUDA (sm_90a) only -- there is no CPU fallback" % what)


def pose_is_f32(cam_E):
    """np.dot(cam_E, [pts 1]) stays in float32 for a float32 pose; every other pose is applied in float64"""
    return np.asarray(cam_E).dtype == np.float32


def vox2pix_into(pix, fov, pix_z, cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id,
                 voxel_range=None):
    """vox2pix into caller-owned CUDA buffers (no allocation): pix int64 (N, P, 2), fov bool (N, P), pix_z: N values
    of the pose's precision (float32 for a float32 pose, else float64; any buffer of that many bytes).  Enqueued on
    the current stream of pix's device.  voxel_range=(v0, n): only voxels [v0, v0 + n) of the grid's C order (an
    X-slab), written to buffers of n voxels -- that slice of the whole grid's result (`occd_vox2pix_range_fwd`).
    pix and pix_z may be None: a FOV mask alone, the same bytes, without the (N, P, 2) index scratch."""
    if not 0 <= int(pattern_id) < len(PIXEL_PATTERNS):
        raise IndexError("pattern_id out of range")        # the reference indexes the same 9-entry list
    X, Y, Z = (int(v) for v in volume_dims(vox_origin, voxel_size, scene_size))
    f32_pose = pose_is_f32(cam_E)
    E = np.ascontiguousarray(np.asarray(cam_E).astype(np.float32 if f32_pose else np.float64))
    k32 = np.ascontiguousarray(np.asarray(cam_k).astype(np.float32))         # fusion.py:331 intr.astype(float32)
    o32 = np.ascontiguousarray(np.asarray(vox_origin).astype(np.float32))    # fusion.py:205
    if E.shape != (4, 4) or k32.shape != (3, 3) or o32.shape != (3,):
        raise ValueError("vox2pix: cam_E must be 4x4, cam_k 3x3, vox_origin (3,)")
    pat = np.ascontiguousarray(np.asarray(PIXEL_PATTERNS[int(pattern_id)], dtype=np.int32))
    P, N = len(pat), X * Y * Z
    if voxel_range is not None:
        v0, N = (int(v) for v in voxel_range)
        if not (v0 >= 0 and N >= 1 and v0 + N <= X * Y * Z):
            raise ValueError("vox2pix_into: voxel_range (%d, %d) is not inside the %d-voxel grid" % (v0, N, X * Y * Z))
    if ((pix is not None and (tuple(pix.shape) != (N, P, 2) or pix.dtype != torch.int64 or not pix.is_contiguous()))
            or tuple(fov.shape) != (N, P) or fov.dtype != torch.bool or not fov.is_contiguous()
            or (pix_z is not None and pix_z.numel() * pix_z.element_size() < N * (4 if f32_pose else 8))):
        raise ValueError("vox2pix_into: the buffers do not hold a (%d, %d) index grid" % (N, P))
    args = (E.ctypes.data_as(C.c_void_p), 1 if f32_pose else 0, k32.ctypes.data_as(C.c_void_p),
            o32.ctypes.data_as(C.c_void_p), float(voxel_size), X, Y, Z, int(img_W), int(img_H),
            pat.ctypes.data_as(C.c_void_p), P, None if pix is None else pix.data_ptr(), fov.data_ptr(),
            None if pix_z is None else pix_z.data_ptr())
    if voxel_range is None:
        _lib.check(_lib.lib().occd_vox2pix_fwd(*args, _lib.stream_ptr()), "occd_vox2pix_fwd")
    else:
        _lib.check(_lib.lib().occd_vox2pix_range_fwd(*args, v0, N, _lib.stream_ptr()), "occd_vox2pix_range_fwd")


def vox2pix(cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id, device=None):
    """occdepth.data.utils.helpers.vox2pix on the GPU (see module docstring).  Raises if no CUDA device."""
    dev = torch.device("cuda" if device is None else device)
    _require_cuda(dev, "vox2pix")
    if not 0 <= int(pattern_id) < len(PIXEL_PATTERNS):
        raise IndexError("pattern_id out of range")
    X, Y, Z = (int(v) for v in volume_dims(vox_origin, voxel_size, scene_size))
    P, N = len(PIXEL_PATTERNS[int(pattern_id)]), X * Y * Z
    with torch.cuda.device(dev):
        pix = torch.empty(N, P, 2, dtype=torch.int64, device=dev)
        fov = torch.empty(N, P, dtype=torch.bool, device=dev)
        pix_z = torch.empty(N, dtype=torch.float32 if pose_is_f32(cam_E) else torch.float64, device=dev)
        vox2pix_into(pix, fov, pix_z, cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id)
    return pix, fov, pix_z


IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)     # kitti_dataset.py:167-169


def normalize_rgb(img_u8, img_H, img_W, mean=IMAGENET_MEAN, std=IMAGENET_STD, device=None):
    """The datasets' image pre-processing on the GPU: uint8 RGB (H0, W0, 3) array / tensor (host or device) ->
    float32 (3, img_H, img_W) CUDA tensor equal, bit for bit, to
    `normalize_rgb((np.array(img, np.float32) / 255.0)[:img_H, :img_W])` of kitti_dataset.py:376-402
    (ToTensor + Normalize).  The host->device copy is the uint8 image (4x smaller than the float tensor)."""
    dev = torch.device("cuda" if device is None else device)
    _require_cuda(dev, "normalize_rgb")
    t = torch.as_tensor(np.asarray(img_u8) if not isinstance(img_u8, torch.Tensor) else img_u8)
    if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError("normalize_rgb: expected a uint8 (H, W, 3) RGB image")
    t = t.contiguous().to(dev, non_blocking=True)
    H0, W0 = int(t.shape[0]), int(t.shape[1])
    m32 = np.ascontiguousarray(np.asarray(mean, dtype=np.float32))
    s32 = np.ascontiguousarray(np.asarray(std, dtype=np.float32))
    with torch.cuda.device(dev):
        out = torch.empty(3, int(img_H), int(img_W), dtype=torch.float32, device=dev)
        rc = _lib.lib().occd_normalize_rgb_u8(t.data_ptr(), out.data_ptr(), H0, W0, int(img_H), int(img_W),
                                              m32.ctypes.data_as(C.c_void_p), s32.ctypes.data_as(C.c_void_p),
                                              _lib.stream_ptr())
        _lib.check(rc, "occd_normalize_rgb_u8")
    return out


def stage_rgb_u8(imgs_u8, out, out_dtype, img_H, img_W, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """`normalize_rgb` of n images written straight into a channels-last buffer: imgs_u8 a CUDA uint8 (n, H0, W0, 3)
    tensor (any image / row strides, pixels 3 contiguous bytes), out a CUDA tensor [n, ..., img_H, img_W, cstride] of
    the activation type `out_dtype` (_lib.DTYPE_F32: TF32 values, _lib.DTYPE_BF16).  Bit for bit
    `occd_planar_to_cl(normalize_rgb(image))`, pad channels zero (`occd_stage_rgb_u8_cl`); enqueued on the current
    stream, no allocation."""
    if not (imgs_u8.is_cuda and imgs_u8.dtype == torch.uint8 and imgs_u8.dim() == 4 and imgs_u8.shape[3] == 3
            and imgs_u8.stride(3) == 1 and imgs_u8.stride(2) == 3):
        raise ValueError("stage_rgb_u8: expected a CUDA uint8 (n, H, W, 3) tensor with 3-byte pixels")
    n, H0, W0 = (int(v) for v in imgs_u8.shape[:3])
    want_dt = {_lib.DTYPE_F32: torch.float32, _lib.DTYPE_BF16: torch.bfloat16}.get(int(out_dtype))
    if not (out.is_cuda and out.dtype == want_dt and out.is_contiguous()
            and out.numel() == n * img_H * img_W * out.shape[-1]):
        raise ValueError("stage_rgb_u8: out must be a contiguous CUDA tensor [n, ..., H, W, cstride]")
    m32 = np.ascontiguousarray(np.asarray(mean, dtype=np.float32))
    s32 = np.ascontiguousarray(np.asarray(std, dtype=np.float32))
    rc = _lib.lib().occd_stage_rgb_u8_cl(imgs_u8.data_ptr(), imgs_u8.stride(0), imgs_u8.stride(1), n, H0, W0,
                                         int(img_H), int(img_W), m32.ctypes.data_as(C.c_void_p),
                                         s32.ctypes.data_as(C.c_void_p), out.data_ptr(), int(out_dtype),
                                         int(out.shape[-1]), _lib.stream_ptr())
    _lib.check(rc, "occd_stage_rgb_u8_cl")


def stage_camera_u8(imgs_u8, out, out_dtype, img_H, img_W, pixel_format="rgb", maps=None, mean=IMAGENET_MEAN,
                    std=IMAGENET_STD):
    """`stage_rgb_u8` of the images cameras and video decoders deliver, bit for bit what OpenCV makes of them on the
    host first (`occd_stage_camera_u8_cl`):
      pixel_format "rgb" / "bgr": imgs_u8 a CUDA uint8 (n, H0, W0, 3) tensor with 3-byte pixels (cv2.COLOR_BGR2RGB);
                   "nv12": a CUDA uint8 (n, H0 * 3 / 2, W0) tensor, OpenCV's NV12 layout (the luma rows, then the
                   interleaved U, V rows; rows of one stride, H0 and W0 even), converted as cv2.COLOR_YUV2RGB_NV12.
      maps: None (the top-left img_H x img_W crop) or a CUDA float32 (n, 2, img_H, img_W) tensor of source x, y per
            output pixel, each image's maps contiguous: the converted images are rectified as
            cv2.remap(rgb, maps[i, 0], maps[i, 1], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT) does.
    Enqueued on the current stream, no allocation."""
    fmt = _lib.PIXEL_FORMATS.get(pixel_format)
    if fmt is None:
        raise ValueError("stage_camera_u8: pixel_format must be one of %s, got %r"
                         % (sorted(_lib.PIXEL_FORMATS), pixel_format))
    if not (imgs_u8.is_cuda and imgs_u8.dtype == torch.uint8):
        raise ValueError("stage_camera_u8: expected a CUDA uint8 tensor")
    if fmt == _lib.PIX_NV12:
        if not (imgs_u8.dim() == 3 and imgs_u8.stride(2) == 1 and imgs_u8.shape[1] % 3 == 0):
            raise ValueError("stage_camera_u8: an NV12 batch is a uint8 (n, H0 * 3 / 2, W0) tensor with 1-byte pixels")
        H0 = int(imgs_u8.shape[1]) * 2 // 3
        uv_offset = H0 * imgs_u8.stride(1)
    else:
        if not (imgs_u8.dim() == 4 and imgs_u8.shape[3] == 3 and imgs_u8.stride(3) == 1 and imgs_u8.stride(2) == 3):
            raise ValueError("stage_camera_u8: expected a uint8 (n, H, W, 3) tensor with 3-byte pixels")
        H0, uv_offset = int(imgs_u8.shape[1]), 0
    n, W0 = int(imgs_u8.shape[0]), int(imgs_u8.shape[2])
    want_dt = {_lib.DTYPE_F32: torch.float32, _lib.DTYPE_BF16: torch.bfloat16}.get(int(out_dtype))
    if not (out.is_cuda and out.dtype == want_dt and out.is_contiguous()
            and out.numel() == n * img_H * img_W * out.shape[-1]):
        raise ValueError("stage_camera_u8: out must be a contiguous CUDA tensor [n, ..., H, W, cstride]")
    map_ptr, map_stride = None, 0
    if maps is not None:
        if not (maps.is_cuda and maps.dtype == torch.float32 and tuple(maps.shape) == (n, 2, img_H, img_W)
                and maps[0].is_contiguous() and maps.device == imgs_u8.device):
            raise ValueError("stage_camera_u8: maps must be a CUDA float32 (%d, 2, %d, %d) tensor on the images' "
                             "device, each image's contiguous" % (n, img_H, img_W))
        map_ptr, map_stride = maps.data_ptr(), maps.stride(0)
    m32 = np.ascontiguousarray(np.asarray(mean, dtype=np.float32))
    s32 = np.ascontiguousarray(np.asarray(std, dtype=np.float32))
    rc = _lib.lib().occd_stage_camera_u8_cl(imgs_u8.data_ptr(), fmt, imgs_u8.stride(0), imgs_u8.stride(1), uv_offset,
                                            n, H0, W0, int(img_H), int(img_W), map_ptr, map_stride,
                                            m32.ctypes.data_as(C.c_void_p), s32.ctypes.data_as(C.c_void_p),
                                            out.data_ptr(), int(out_dtype), int(out.shape[-1]), _lib.stream_ptr())
    _lib.check(rc, "occd_stage_camera_u8_cl")


NYU_DEPTH_SCALE, NYU_MAX_DEPTH = 8000.0, 10.0     # nyu_dataset.py:42-48


def depth_u16_to_f32(depth_u16, out, divisor=NYU_DEPTH_SCALE, max_depth=NYU_MAX_DEPTH):
    """NYU's `load_depth` of a decoded uint16 depth PNG into a CUDA float32 tensor of the same element count:
    float32(depth / divisor) (float64 division), clamped to [0, max_depth] (`occd_depth_u16_to_f32`); enqueued on the
    current stream, no allocation."""
    if not (depth_u16.is_cuda and depth_u16.dtype == torch.uint16 and depth_u16.is_contiguous()):
        raise ValueError("depth_u16_to_f32: expected a contiguous CUDA uint16 tensor")
    if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.numel() == depth_u16.numel()):
        raise ValueError("depth_u16_to_f32: out must be a contiguous CUDA float32 tensor of the same size")
    rc = _lib.lib().occd_depth_u16_to_f32(depth_u16.data_ptr(), out.data_ptr(), depth_u16.numel(), float(divisor),
                                          float(max_depth), _lib.stream_ptr())
    _lib.check(rc, "occd_depth_u16_to_f32")
