"""Numpy restatement of what the reference's visualisation scripts build from a prediction
(scripts/visualization/kitti_vis_pred.py:9-32 and 69-89, kitti_vis_pred_batch.py:92-106, NYU_vis_pred.py:67-78): the
voxel-centre grid, the class attached to every row, the FOV split and the rows with 0 < class < 255.  The scripts
import mayavi / open3d and cannot be imported; `tests/test_voxel_list_host.py` checks this restatement against a
line-by-line transcription of them.  Everything is float64, as there; `rows32` rounds to the float32 the device writes.
"""
import numpy as np


def grid_coords(dims, resolution):
    """get_grid_coords: float64 [D1*D0*D2, 3].  The axes are meshed x-y (`np.meshgrid`'s default "xy" indexing, so
    row (i*D0 + j)*D2 + k pairs g_xx[j] with g_yy[i]), scaled to `idx * resolution + resolution / 2`, and the first
    two columns are swapped afterwards: the row holds the centre of (i, j, k), i < D1, j < D0.  Only for D0 == D1 is
    that the voxel whose class `voxels.reshape(-1)` puts on the same row -- the scripts always call it that way.  No
    origin is added."""
    D0, D1, D2 = (int(d) for d in dims)
    i, j, k = np.indices((D1, D0, D2))
    idx = np.stack([i.reshape(-1), j.reshape(-1), k.reshape(-1)], axis=1).astype(np.float64)
    return idx * resolution + resolution / 2


def centres(shape, resolution, origin=None):
    """float64 centres of the voxels of a C-ordered [X, Y, Z] grid, row = flat index; `origin` added afterwards"""
    idx = np.stack([a.reshape(-1) for a in np.indices(tuple(int(s) for s in shape))], axis=1).astype(np.float64)
    c = idx * resolution + resolution / 2
    return c if origin is None else c + np.asarray(origin, dtype=np.float64)


def select(y_pred, fov_mask=None, empty=0, ignore=255):
    """(flat indices of the occupied voxels inside the FOV, outside it), ascending: boolean indexing's order"""
    flat = np.asarray(y_pred).reshape(-1)
    occ = (flat > empty) & (flat < ignore)
    if fov_mask is None:
        return np.flatnonzero(occ), np.zeros(0, dtype=np.int64)
    m = np.asarray(fov_mask).reshape(-1).astype(bool)
    return np.flatnonzero(occ & m), np.flatnonzero(occ & ~m)


def kitti_rows(y_pred, fov_mask, voxel_size=0.2):
    """(fov_voxels, outfov_voxels) of kitti_vis_pred.py's draw(): float64 [n, 4] rows [x, y, z, class]"""
    y_pred = np.asarray(y_pred)
    grid = np.hstack([centres(y_pred.shape, voxel_size), y_pred.reshape(-1, 1).astype(np.float64)])
    i_in, i_out = select(y_pred, fov_mask)
    return grid[i_in], grid[i_out]


def nyu_rows(y_pred, voxel_size=0.08):
    """occupied_voxels of NYU_vis_pred.py's draw(): the rows of the map with its last two axes exchanged"""
    return kitti_rows(np.moveaxis(np.asarray(y_pred), [0, 1, 2], [0, 2, 1]), None, voxel_size)[0]


def voxel_list(y_pred, fov_mask=None, voxel_size=None, origin=None, index0=0, n_hist=64, empty=0, ignore=255):
    """what occd_occupied_voxels writes for one frame, untruncated: dict of count (2,), hist (n_hist,), index int32,
    cls uint16, xyz float32 (None without voxel_size); `index0` offsets the indices into a larger grid with the same
    Y, Z (coordinates follow)"""
    y_pred = np.asarray(y_pred)
    X, Y, Z = y_pred.shape
    i_in, i_out = select(y_pred, fov_mask, empty, ignore)
    order = np.concatenate([i_in, i_out]).astype(np.int64)
    cls = y_pred.reshape(-1)[order].astype(np.uint16)
    hist = np.bincount(cls[cls < n_hist], minlength=n_hist).astype(np.int64)
    gi = order + int(index0)
    xyz = None
    if voxel_size is not None:
        idx = np.stack([gi // (Y * Z), gi // Z % Y, gi % Z], axis=1).astype(np.float64)
        c = idx * voxel_size + voxel_size / 2
        if origin is not None:
            c = c + np.asarray(origin, dtype=np.float64)
        xyz = c.astype(np.float32)
    return dict(count=np.array([len(i_in), len(i_out)], dtype=np.int64), hist=hist, index=gi.astype(np.int32),
                cls=cls, xyz=xyz)


def rows32(rows):
    return np.asarray(rows).astype(np.float32)
