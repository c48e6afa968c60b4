"""The occupied voxels of a class map as an ordered list, built on the device.

Every consumer of a prediction the reference has turns the dense map into rows `[x, y, z, class]` of the occupied
voxels first: its visualisation scripts (scripts/visualization/kitti_vis_pred.py:69-89, kitti_vis_pred_batch.py,
NYU_vis_pred.py) mesh the voxel centres with `get_grid_coords`, attach the class, split the rows with `fov_mask_1` and
keep those with `0 < class < 255` -- numpy passes over every voxel, after the whole map was read back.
`occupied_voxels` does the selection in three launches (`occd_occupied_voxels`) and leaves the rows on the device in
numpy's order (in-FOV voxels first, each group in ascending flat index), so a caller reads back the occupied rows only.

    vl = occupied_voxels(model.predict_classes(batch), fov_mask, voxel_size=0.2)
    fov_voxels, outfov_voxels = vl.rows()          # the two [n, 4] arrays the KITTI scripts draw

A voxel's coordinates are the centre of its own (x, y, z) index: float32(idx * voxel_size + voxel_size / 2), formed in
float64 as numpy does.  For a grid with X == Y -- the only way the scripts call it -- these are the rows of
`get_grid_coords([X, Y, Z], voxel_size)`; `vox_origin`, when given, is added in float64 before the rounding (the
scripts themselves stay in the grid's frame and move the camera instead).  NYU_vis_pred.py lists the voxels of
`np.moveaxis(y_pred, [0, 1, 2], [0, 2, 1])`: pass `class_map.transpose(-1, -2).contiguous()` for its rows.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

HIST_BINS = 64          # class ids counted by the histogram (the class LUT's cap); larger ids are listed, not counted


class VoxelList:
    """Device tensors of one `occupied_voxels` call over B frames of N voxels, `capacity` rows per frame:
      count int32 [B, 2]   occupied voxels inside / outside the FOV (the true counts, also when truncated)
      hist  int32 [B, 64]  occupied voxels per class id
      index int32 [B, capacity]   flat voxel index     cls uint16 [B, capacity]
      xyz   float32 [B, capacity, 3] voxel centres, or None when no voxel_size was given
    Row r of frame b is valid for r < min(capacity, count[b].sum()); the rest holds whatever it held before.
    Nothing here synchronises with the host except `counts()`, `truncated` and `rows()`."""

    def __init__(self, B, N, capacity, with_xyz, device):
        self.B, self.N, self.capacity = B, N, capacity
        self.count = torch.zeros(B, 2, dtype=torch.int32, device=device)
        self.hist = torch.zeros(B, HIST_BINS, dtype=torch.int32, device=device)
        self.index = torch.empty(B, capacity, dtype=torch.int32, device=device)
        self.cls = torch.empty(B, capacity, dtype=torch.uint16, device=device)
        self.xyz = torch.empty(B, capacity, 3, dtype=torch.float32, device=device) if with_xyz else None
        # the kernels' tile counts: one (inside, outside) uint32 pair per tile, held as one int64 (8-byte aligned)
        self.work = torch.empty(_lib.voxel_work_len(B, N) // 2, dtype=torch.int64, device=device)
        self._counts = None

    def counts(self):
        """int64 numpy [B, 2]: occupied voxels inside / outside the FOV (one device->host read, cached)"""
        if self._counts is None:
            self._counts = self.count.cpu().numpy().astype(np.int64)
        return self._counts

    @property
    def truncated(self):
        """True when some frame holds more occupied voxels than `capacity` rows (reads the counts)"""
        return bool((self.counts().sum(1) > self.capacity).any())

    def split(self, b=0):
        """(rows inside the FOV, rows outside) of frame b that were written: n_in + n_out <= capacity"""
        n_in, n_out = (int(v) for v in self.counts()[b])
        n_in_w = min(n_in, self.capacity)
        return n_in_w, min(n_out, self.capacity - n_in_w), n_in

    def rows(self, b=0):
        """(fov_voxels, outfov_voxels) of frame b: float32 numpy [n, 4] rows `[x, y, z, class]`, the arrays the
        visualisation scripts build (theirs are float64; these are those values rounded to float32).  Without a FOV
        mask every row is in the first array.  Reads back the written rows only."""
        if self.xyz is None:
            raise ValueError("VoxelList.rows: no coordinates were computed (pass voxel_size to occupied_voxels)")
        n_in, n_out, first_out = self.split(b)
        out = []
        for lo, n in ((0, n_in), (first_out, n_out)):
            r = np.empty((n, 4), dtype=np.float32)
            r[:, :3] = self.xyz[b, lo:lo + n].cpu().numpy()
            r[:, 3] = self.cls[b, lo:lo + n].cpu().numpy()
            out.append(r)
        return tuple(out)


def _mask_bytes(fov_mask, B, N, dev):
    m = fov_mask
    if not isinstance(m, torch.Tensor):
        m = torch.from_numpy(np.ascontiguousarray(m))
    if m.dtype not in (torch.bool, torch.uint8):
        raise TypeError("occupied_voxels: fov_mask must be bool (or its uint8 bytes), got %s" % m.dtype)
    if m.numel() != B * N:
        raise ValueError("occupied_voxels: fov_mask holds %d values, the class map %d" % (m.numel(), B * N))
    if not m.is_contiguous():
        raise ValueError("occupied_voxels: fov_mask must be contiguous")
    if m.device != dev:
        if m.is_cuda:
            raise ValueError("occupied_voxels: class_map on %s, fov_mask on %s" % (dev, m.device))
        m = m.to(dev, non_blocking=True)
    return m


def occupied_voxels(class_map, fov_mask=None, *, voxel_size=None, vox_origin=None, capacity=None, empty=0, ignore=255,
                    index0=0, out=None):
    """The ordered occupied-voxel list of `class_map` (CUDA uint16 [B, X, Y, Z] or [X, Y, Z], contiguous: what
    predict_classes / class_map return, remapped or not) -> VoxelList.  Enqueued on the current stream; no host
    synchronisation.

    fov_mask: bool [B, N] (any shape of B*N values; host arrays are copied over), e.g. a frame's `fov_mask_1`; None
              lists every occupied voxel as inside.
    voxel_size: edge of a voxel in metres; given, the voxel centres are written too (see the module docstring).
    vox_origin: 3 values added to the centres (default: none, the grid's own frame).
    capacity: rows per frame (default N: never truncates).  A frame with more occupied voxels keeps its first
              `capacity` rows in order; `count` still holds the true counts and `truncated` tells.
    empty, ignore: a voxel is occupied when empty < class < ignore.
    index0: flat index of the map's first voxel inside a larger grid (an X-slab: x_lo * Y * Z); indices and
            coordinates are those of the larger grid.
    out: a VoxelList of an earlier call with the same B, N and capacity, whose tensors are overwritten (a serving
         loop then allocates nothing per frame)."""
    if not (isinstance(class_map, torch.Tensor) and class_map.is_cuda and class_map.dtype == torch.uint16):
        raise TypeError("occupied_voxels: class_map must be a CUDA uint16 tensor (there is no CPU fallback)")
    if class_map.dim() == 3:
        class_map = class_map.unsqueeze(0)
    if class_map.dim() != 4 or class_map.numel() == 0 or not class_map.is_contiguous():
        raise ValueError("occupied_voxels: class_map must be a contiguous, non-empty [B, X, Y, Z] tensor")
    B, X, Y, Z = (int(v) for v in class_map.shape)
    N = X * Y * Z
    dev = class_map.device
    cap = N if capacity is None else int(capacity)
    if cap < 0:
        raise ValueError("occupied_voxels: capacity must be >= 0")
    with_xyz = voxel_size is not None
    if vox_origin is not None and not with_xyz:
        raise ValueError("occupied_voxels: vox_origin without voxel_size")
    origin = None
    if vox_origin is not None:
        origin = np.ascontiguousarray(np.asarray(vox_origin, dtype=np.float64).reshape(-1))
        if origin.shape != (3,):
            raise ValueError("occupied_voxels: vox_origin must hold 3 values")
    with torch.cuda.device(dev):
        mask = None if fov_mask is None else _mask_bytes(fov_mask, B, N, dev)
        if out is None:
            out = VoxelList(B, N, cap, with_xyz, dev)
        elif ((out.B, out.N, out.capacity) != (B, N, cap) or (out.xyz is not None) != with_xyz
              or out.count.device != dev):
            raise ValueError("occupied_voxels: `out` was made for another shape, capacity or device")
        out._counts = None
        rc = _lib.lib().occd_occupied_voxels(
            class_map.data_ptr(), None if mask is None else mask.data_ptr(), B, X, Y, Z, int(index0), int(empty),
            int(ignore), HIST_BINS, cap, out.count.data_ptr(), out.hist.data_ptr(), out.index.data_ptr(),
            out.cls.data_ptr(), None if out.xyz is None else out.xyz.data_ptr(),
            float(voxel_size) if with_xyz else 0.0, None if origin is None else origin.ctypes.data_as(C.c_void_p),
            out.work.data_ptr(), 2 * out.work.numel(), _lib.stream_ptr())
        _lib.check(rc, "occd_occupied_voxels")
    return out
