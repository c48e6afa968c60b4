"""Scene maps restated in numpy: the reference the tests hold `occd_scene_map_integrate`, `occd_scene_map_shift` and
`occd_scene_map_mark_unobserved` to.

The index math is float64 element-wise, in the order the header states (no fused multiply-add in numpy), so frame
indices and observed flags match the kernel bit for bit.  The accumulation is float32 with numpy's `log`, which may
differ from the device's `logf` in the last bits: that step alone is compared with a tolerance."""
import numpy as np


def plane_layout(shape, axes):
    """(GX, GY, GZ) and the element strides (x, y, z) of one class plane of storage shape (D0, D1, D2)"""
    D0, D1, D2 = (int(v) for v in shape)
    if axes == "xyz":
        return (D0, D1, D2), (D1 * D2, D2, 1)
    if axes == "xzy":
        return (D0, D2, D1), (D1 * D2, 1, D2)
    raise ValueError(axes)


def frame_index(R, origin, voxel, dims, grid_origin, grid_voxel, grid_dims):
    """float64 frame indices f [3, MX, MY, MZ] of every map voxel and the bool `inside` [MX, MY, MZ]"""
    idx = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in dims], indexing="ij")
    c = [(idx[a] + 0.5) * voxel + origin[a] for a in range(3)]
    f = np.empty((3,) + tuple(dims), np.float64)
    for r in range(3):
        q = ((R[r, 0] * c[0] + R[r, 1] * c[1]) + R[r, 2] * c[2]) + R[r, 3]
        f[r] = np.floor((q - grid_origin[r]) / grid_voxel)
    inside = np.ones(tuple(dims), bool)
    for r in range(3):
        inside &= (f[r] >= 0) & (f[r] < grid_dims[r])
    return f, inside


def integrate(acc, count, origin, voxel, probs, T, grid_origin, grid_voxel, axes="xyz", fov_mask=None,
              min_prob=1e-3):
    """one frame into acc float32 [C, MX, MY, MZ] and count int32 [MX, MY, MZ], in place; probs float16
    [C, D0, D1, D2]; returns the bool mask of the voxels written"""
    R = np.linalg.inv(np.asarray(T, np.float64))
    C = probs.shape[0]
    G, s = plane_layout(probs.shape[1:], axes)
    f, obs = frame_index(R, np.asarray(origin, np.float64), float(voxel), count.shape,
                         np.asarray(grid_origin, np.float64), float(grid_voxel), G)
    fi = np.where(obs[None], f, 0).astype(np.int64)
    off = fi[0] * s[0] + fi[1] * s[1] + fi[2] * s[2]
    if fov_mask is not None:
        obs &= np.asarray(fov_mask).reshape(-1).astype(bool)[off]
    p = probs.reshape(C, -1)[:, off[obs]].astype(np.float32)
    ok = ~np.isnan(p).any(0)
    sel = np.flatnonzero(obs)[ok]
    obs = np.zeros_like(obs)
    obs.reshape(-1)[sel] = True
    a = acc.reshape(C, -1)
    a[:, sel] = a[:, sel] + np.log(np.maximum(p[:, ok], np.float32(min_prob)))
    count.reshape(-1)[sel] += 1
    return obs


def shift(a, d):
    """out[..., idx] = a[..., idx + d] over the last three axes, 0 where idx + d leaves the grid"""
    out = np.zeros_like(a)
    src, dst = [], []
    for n, s in zip(a.shape[-3:], d):
        lo, hi = max(0, -s), min(n, n - s)
        if lo >= hi:
            return out
        dst.append(slice(lo, hi))
        src.append(slice(lo + s, hi + s))
    out[(Ellipsis,) + tuple(dst)] = a[(Ellipsis,) + tuple(src)]
    return out


def mark_unobserved(class_map, count, unknown=255):
    return np.where(count == 0, np.uint16(unknown), class_map).astype(np.uint16)
