"""Host side of the occupied-voxel list: the oracle's selection and coordinates against a transcription of what the
reference's visualisation scripts compute (kitti_vis_pred.py / kitti_vis_pred_batch.py / NYU_vis_pred.py), and the
argument checks of occd_occupied_voxels that need no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from occdepth_b200 import _build, _lib
from oracle import voxel_list as OV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KITTI, NYU = (256, 256, 32), (60, 36, 60)


# ---- the scripts, step by step ---------------------------------------------------------------------------------------
def script_grid_coords(dims, resolution):
    g_xx, g_yy, g_zz = (np.arange(0, d + 1) for d in dims)
    xx, yy, zz = np.meshgrid(g_xx[:-1], g_yy[:-1], g_zz[:-1])
    coords_grid = np.array([xx.flatten(), yy.flatten(), zz.flatten()]).T.astype(np.float64)
    coords_grid = (coords_grid * resolution) + resolution / 2
    temp = np.copy(coords_grid)
    temp[:, 0] = coords_grid[:, 1]
    temp[:, 1] = coords_grid[:, 0]
    return np.copy(temp)


def script_kitti(voxels, fov_mask, voxel_size=0.2):
    grid_coords = script_grid_coords([voxels.shape[0], voxels.shape[1], voxels.shape[2]], voxel_size)
    grid_coords = np.vstack([grid_coords.T, voxels.reshape(-1)]).T
    fov_grid_coords = grid_coords[fov_mask, :]
    outfov_grid_coords = grid_coords[~fov_mask, :]
    fov_voxels = fov_grid_coords[(fov_grid_coords[:, 3] > 0) & (fov_grid_coords[:, 3] < 255)]
    outfov_voxels = outfov_grid_coords[(outfov_grid_coords[:, 3] > 0) & (outfov_grid_coords[:, 3] < 255)]
    return fov_voxels, outfov_voxels


def script_nyu(voxels, voxel_size=0.08):
    grid_coords = script_grid_coords([voxels.shape[0], voxels.shape[2], voxels.shape[1]], voxel_size)
    grid_coords = np.vstack((grid_coords.T, np.moveaxis(voxels, [0, 1, 2], [0, 2, 1]).reshape(-1))).T
    return grid_coords[(grid_coords[:, 3] > 0) & (grid_coords[:, 3] < 255)]


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.ascontiguousarray(a).tobytes() == \
        np.ascontiguousarray(b).tobytes()


def _map(shape, n_classes, seed, occupied=0.05):
    g = np.random.default_rng(seed)
    y = g.integers(1, n_classes, size=shape).astype(np.uint16)
    y[g.random(shape) > occupied] = 0
    y.reshape(-1)[g.integers(0, y.size, 50)] = 255
    return y, g.random(y.size) < 0.4


# ---- 1. the oracle against the scripts --------------------------------------------------------------------------------
@pytest.mark.parametrize("dims,res", [(KITTI, 0.2), ((60, 60, 36), 0.08), ((5, 3, 4), 0.2), ((3, 5, 2), 0.08)])
def test_grid_coords(dims, res):
    want = script_grid_coords(list(dims), res)
    assert _same(OV.grid_coords(dims, res), want)
    if dims[0] == dims[1]:                       # the only grids the scripts mesh: row = the voxel's own centre
        assert _same(OV.centres(dims, res), want)


@pytest.mark.parametrize("inv", [False, True])
def test_kitti_rows(inv):
    y, mask = _map(KITTI, 20, 0)
    if inv:                                      # the submission writer's remap, generate_kitti_submission.py:79
        lut = np.random.default_rng(1).permutation(np.arange(1, 100))[:20]
        lut[0] = 0
        y = np.where(y == 255, 255, lut[np.minimum(y, 19)]).astype(np.uint16)
    want = script_kitti(y, mask)
    got = OV.kitti_rows(y, mask)
    assert _same(got[0], want[0]) and _same(got[1], want[1])
    assert len(want[0]) > 1000 and len(want[1]) > 1000
    # the device's arrays are those rows in float32, in-FOV first
    vl = OV.voxel_list(y, mask, voxel_size=0.2)
    rows = np.concatenate([vl["xyz"], vl["cls"][:, None].astype(np.float32)], axis=1)
    assert _same(rows, OV.rows32(np.concatenate(want)))
    assert vl["count"].tolist() == [len(want[0]), len(want[1])]
    assert vl["hist"].sum() == (vl["cls"] < 64).sum() and vl["index"].dtype == np.int32


def test_without_mask_and_nyu_rows():
    y, _ = _map(NYU, 12, 2, occupied=0.3)
    want = script_nyu(y)
    assert _same(OV.nyu_rows(y), want)
    # the same rows from the list of the transposed map, which is how a caller gets them from the device
    yt = np.ascontiguousarray(np.moveaxis(y, [0, 1, 2], [0, 2, 1]))
    vl = OV.voxel_list(yt, None, voxel_size=0.08)
    assert vl["count"].tolist() == [len(want), 0]
    assert _same(np.concatenate([vl["xyz"], vl["cls"][:, None].astype(np.float32)], axis=1), OV.rows32(want))
    # the map as predicted: the same voxels, each with its own centre
    v0 = OV.voxel_list(y, None, voxel_size=0.08)
    x, yy, z = np.unravel_index(v0["index"], NYU)
    assert _same(v0["xyz"], (np.stack([x, yy, z], 1) * 0.08 + 0.08 / 2).astype(np.float32))


def test_index0_is_a_window_of_the_whole_grid():
    y, mask = _map((16, 6, 5), 12, 3, occupied=0.4)
    whole = OV.voxel_list(y, mask, voxel_size=0.2, origin=[0, -25.6, -2])
    parts = [OV.voxel_list(y[lo:hi], mask.reshape(16, -1)[lo:hi], voxel_size=0.2, origin=[0, -25.6, -2],
                           index0=lo * 30) for lo, hi in ((0, 4), (4, 12), (12, 16))]
    n_in = [int(p["count"][0]) for p in parts]
    for k in ("index", "cls", "xyz"):
        cat = np.concatenate([p[k][:n] for p, n in zip(parts, n_in)] + [p[k][n:] for p, n in zip(parts, n_in)])
        assert _same(cat, whole[k]), k


# ---- 2. the C entry point's argument checks ----------------------------------------------------------------------------
def test_header_and_binding_agree_on_the_workspace():
    src = open(os.path.join(ROOT, "include", "occdepth_b200.h")).read()
    assert int(re.search(r"#define OCCD_VOXEL_TILE (\d+)", src).group(1)) == _lib.VOXEL_TILE
    assert _lib.voxel_work_len(2, 2049) == 2 * 2 * 2 and _lib.voxel_work_len(1, 2048) == 2


def test_argument_validation_without_gpu():
    _build.build()
    L = _lib.lib()
    buf = (C.c_uint64 * 64)()
    p = C.addressof(buf)

    def call(class_map=p, fov=None, B=1, X=4, Y=4, Z=4, index0=0, empty=0, ignore=255, n_classes=20, cap=8, count=p,
             hist=p, index=p, cls=p, xyz=None, voxel_size=0.2, origin=None, work=p, work_len=2):
        return L.occd_occupied_voxels(class_map, fov, B, X, Y, Z, index0, empty, ignore, n_classes, cap, count, hist,
                                      index, cls, xyz, voxel_size, origin, work, work_len, None)
    for bad in (dict(class_map=None), dict(count=None), dict(hist=None), dict(work=None), dict(index=None),
                dict(cls=None), dict(n_classes=65), dict(n_classes=0), dict(B=0), dict(X=-1), dict(Z=0), dict(cap=-1),
                dict(index0=-1), dict(work_len=1), dict(X=2048, Y=2048, Z=1024), dict(empty=-1), dict(ignore=70000),
                dict(xyz=p, voxel_size=0.0), dict(class_map=p + 1), dict(work=p + 4)):
        assert call(**bad) == _lib.ERR_ARG, bad
        assert b"occd_occupied_voxels" in L.occd_last_error()
