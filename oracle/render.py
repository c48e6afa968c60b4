"""Camera views restated in numpy: the reference the tests hold `occd_render_classes` to.

The ray walk of csrc/render.cuh in float64 element-wise numpy, vectorised over pixels, every operation in the
header's order (numpy has no fused multiply-add) and every min / max the same plain comparison, so class, depth and
index match the kernel bit for bit.  It runs on any subset of pixels: the rays are independent."""
import numpy as np

from .scene_map import plane_layout  # noqa: F401  (the same storage orders)


def camera(E, K):
    """the 12 float64 values of one camera: M = R^-1 K^-1 row-major, then o = -R^-1 t, from inverse(E)"""
    Ei = np.linalg.inv(np.asarray(E, np.float64))
    M = Ei[:3, :3] @ np.linalg.inv(np.asarray(K, np.float64))
    return np.concatenate([M.reshape(-1), Ei[:3, 3]])


def render(cmap, G, s, origin, voxel, cam, u, v, empty=0, ignore=255, near=0.0, far=np.inf):
    """(cls uint16, depth float32, index int32) of pixels (u, v) (equal-length int arrays) of camera `cam` (12
    float64) through one map `cmap` (uint16, read flat at i*s_x + j*s_y + k*s_z)"""
    flat = np.ascontiguousarray(cmap).reshape(-1)
    u = np.asarray(u, np.int64).reshape(-1).astype(np.float64)
    v = np.asarray(v, np.int64).reshape(-1).astype(np.float64)
    n = u.size
    origin = [float(x) for x in origin]
    voxel = float(voxel)
    G = [int(x) for x in G]
    s = [int(x) for x in s]
    cam = np.asarray(cam, np.float64).reshape(-1)
    M, o = cam[:9].reshape(3, 3), [float(x) for x in cam[9:12]]
    cls = np.full(n, empty, np.uint16)
    depth = np.full(n, np.inf, np.float32)
    index = np.full(n, -1, np.int32)

    def btime(a, i, r):
        return ((origin[a] + i.astype(np.float64) * voxel) - o[a]) * r

    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d = np.stack([(M[a, 0] * u + M[a, 1] * v) + M[a, 2] for a in range(3)])
        zero = d == 0.0
        r = np.where(zero, 0.0, 1.0 / np.where(zero, 1.0, d))
        alive = np.ones(n, bool)
        t_lo = np.full(n, -np.inf)
        t_hi = np.full(n, np.inf)
        for a in range(3):
            hi = origin[a] + float(G[a]) * voxel
            inside = origin[a] <= o[a] and o[a] < hi
            if not inside:
                alive &= ~zero[a]
            ta = btime(a, np.zeros(n, np.int64), r[a])
            tb = btime(a, np.full(n, G[a], np.int64), r[a])
            mn = np.where(ta < tb, ta, tb)
            mx = np.where(ta > tb, ta, tb)
            t_lo = np.where(zero[a], t_lo, np.where(t_lo > mn, t_lo, mn))
            t_hi = np.where(zero[a], t_hi, np.where(t_hi < mx, t_hi, mx))
        t0 = np.where(t_lo > near, t_lo, near)
        t_end = np.where(t_hi < far, t_hi, far)
        alive &= t0 < t_end
        act = np.flatnonzero(alive)
        d, r, t0, t_end = d[:, act], r[:, act], t0[act], t_end[act]
        idx = np.empty((3, act.size), np.int64)
        tn = np.empty((3, act.size))
        for a in range(3):
            f = np.floor(((o[a] + t0 * d[a]) - origin[a]) / voxel)
            f = np.where(f < 0.0, 0.0, f)
            f = np.where(f > float(G[a] - 1), float(G[a] - 1), f)
            idx[a] = f.astype(np.int64)
            tn[a] = np.where(d[a] == 0.0, np.inf, btime(a, idx[a] + (d[a] > 0.0), r[a]))
        step = np.where(d > 0.0, 1, -1)
        t = t0
        for _ in range(G[0] + G[1] + G[2] + 3):
            if act.size == 0:
                break
            off = idx[0] * s[0] + idx[1] * s[1] + idx[2] * s[2]
            c = flat[off].astype(np.int64)
            hit = (c != empty) & (c != ignore)
            cls[act[hit]] = c[hit]
            depth[act[hit]] = t[hit].astype(np.float32)
            index[act[hit]] = off[hit]
            cols = np.arange(act.size)
            a = np.zeros(act.size, np.int64)
            sel = tn[0].copy()
            for b in (1, 2):
                m = tn[b] < sel
                a[m] = b
                sel = np.where(m, tn[b], sel)
            go = ~hit & (sel < t_end)
            t = np.where(t > sel, t, sel)
            idx[a, cols] += step[a, cols]
            ia = idx[a, cols]
            go &= (ia >= 0) & (ia < np.asarray(G)[a])
            for b in range(3):
                m = go & (a == b)
                tn[b, m] = btime(b, idx[b, m] + (step[b, m] > 0), r[b, m])
            act, idx, tn, step, d, r, t, t_end = (act[go], idx[:, go], tn[:, go], step[:, go], d[:, go], r[:, go],
                                                 t[go], t_end[go])
    return cls, depth, index


def render_image(cmap, G, s, origin, voxel, cam, W, H, rows=None, **kw):
    """the [len(rows), W] images of `render` over rows `rows` (default every row) of a W x H view"""
    rows = np.arange(H) if rows is None else np.asarray(rows)
    vv, uu = np.meshgrid(rows, np.arange(W), indexing="ij")
    out = render(cmap, G, s, origin, voxel, cam, uu.reshape(-1), vv.reshape(-1), **kw)
    return tuple(x.reshape(len(rows), W) for x in out)
