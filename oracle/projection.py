"""CPU restatement of the reference's voxel -> pixel projection (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows occdepth/data/utils/helpers.py:94-169 (`vox2pix`) with fusion.py:201-217 (`vox2world`), :518-522
(`rigid_transform`) and :236-343 (`cam2allpixs`), in plain numpy with the reference's dtypes:
voxel centres in float64 then cast to float32; pose applied with np.dot in float64 (so the summation order is
whatever this numpy's BLAS does, exactly as in the reference); intrinsics cast to float32; np.round (half to even);
int64 pixels.  Pinned against the reference itself (numba-compiled) through the fixtures of
tests/test_oracle_vs_reference.py and tests/golden/vox2pix.pt.
"""
import numpy as np

# fusion.py:238-330
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


def vox2pix(cam_E, cam_k, vox_origin, voxel_size, img_W, img_H, scene_size, pattern_id):
    vox_origin = np.asarray(vox_origin)
    vol_bnds = np.zeros((3, 2))                                                    # helpers.py:126-128
    vol_bnds[:, 0] = vox_origin
    vol_bnds[:, 1] = vox_origin + np.array(scene_size)
    vol_dim = np.ceil((vol_bnds[:, 1] - vol_bnds[:, 0]) / voxel_size).copy(order="C").astype(int)   # :131-135
    xv, yv, zv = np.meshgrid(range(vol_dim[0]), range(vol_dim[1]), range(vol_dim[2]), indexing="ij")
    vox = np.concatenate([xv.reshape(1, -1), yv.reshape(1, -1), zv.reshape(1, -1)], 0).astype(int).T
    # fusion.py:201-217: float32 origin and coordinates, float64 scalar voxel size, result stored as float32
    o32 = vox_origin.astype(np.float32)
    c32 = vox.astype(np.float32)
    pts = (o32[None, :].astype(np.float64) + voxel_size * c32.astype(np.float64) + voxel_size * 0.5).astype(np.float32)
    # fusion.py:518-522
    xyz_h = np.hstack([pts, np.ones((len(pts), 1), dtype=np.float32)])
    cam = np.dot(cam_E, xyz_h.T).T[:, :3]
    # fusion.py:331-342
    intr = np.asarray(cam_k).astype(np.float32)
    fx, fy, cx, cy = intr[0, 0], intr[1, 1], intr[0, 2], intr[1, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        xr = np.round(cam[:, 0] * fx / cam[:, 2] + cx)
        yr = np.round(cam[:, 1] * fy / cam[:, 2] + cy)

    def to_int(v):        # int() of the compiled reference: x86 conversion, INT64_MIN for NaN / out of range
        ok = np.isfinite(v) & (v >= -2.0 ** 63) & (v < 2.0 ** 63)
        return np.where(ok, np.where(ok, v, 0).astype(np.int64), np.iinfo(np.int64).min)

    xc, yc = to_int(xr), to_int(yr)
    pat = np.asarray(PIXEL_PATTERNS[pattern_id], dtype=np.int64)
    pix = np.stack([xc[:, None] + pat[None, :, 0], yc[:, None] + pat[None, :, 1]], -1)
    pix_z = cam[:, 2]
    fov = (pix[..., 0] >= 0) & (pix[..., 0] < img_W) & (pix[..., 1] >= 0) & (pix[..., 1] < img_H) & (pix_z[:, None] > 0)
    return pix, fov, pix_z
