"""Soft camera views restated in numpy: the reference the tests hold `occd_render_probs` to.

`walk` is the ray walk of csrc/render.cuh (the one oracle/render.py restates for `occd_render_classes`), vectorised
over pixels, handing each step's voxels to a visitor; tests/test_render_probs_host.py checks that the hard render
built on it equals oracle.render.render bit for bit.  `render_probs` composites float16 class probabilities along it
in float32, element-wise and in the header's order (numpy has no fused multiply-add), so class, depth, opacity and
channels match the kernel bit for bit."""
import numpy as np

from .render import camera, plane_layout  # noqa: F401  (the same cameras and storage orders)


def walk(G, s, origin, voxel, cam, u, v, visit, near=0.0, far=np.inf):
    """Walk pixels (u, v)'s rays: visit(rays, off, t) for the rays still walking (indices into u), their voxels'
    element offsets and float64 entry times, step by step; it returns a bool mask of the rays that stop there"""
    u = np.asarray(u, np.int64).reshape(-1).astype(np.float64)
    v = np.asarray(v, np.int64).reshape(-1).astype(np.float64)
    n = u.size
    origin = [float(x) for x in origin]
    voxel = float(voxel)
    G = [int(x) for x in G]
    s = [int(x) for x in s]
    cam = np.asarray(cam, np.float64).reshape(-1)
    M, o = cam[:9].reshape(3, 3), [float(x) for x in cam[9:12]]

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
            if not (origin[a] <= o[a] and o[a] < hi):
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
            stop = np.asarray(visit(act, off, t), bool)
            cols = np.arange(act.size)
            a = np.zeros(act.size, np.int64)
            sel = tn[0].copy()
            for b in (1, 2):
                m = tn[b] < sel
                a[m] = b
                sel = np.where(m, tn[b], sel)
            go = ~stop & (sel < t_end)
            t = np.where(t > sel, t, sel)
            idx[a, cols] += step[a, cols]
            ia = idx[a, cols]
            go &= (ia >= 0) & (ia < np.asarray(G)[a])
            for b in range(3):
                m = go & (a == b)
                tn[b, m] = btime(b, idx[b, m] + (step[b, m] > 0), r[b, m])
            act, idx, tn, step, d, r, t, t_end = (act[go], idx[:, go], tn[:, go], step[:, go], d[:, go], r[:, go],
                                                 t[go], t_end[go])


def render_hard(cmap, G, s, origin, voxel, cam, u, v, empty=0, ignore=255, near=0.0, far=np.inf):
    """oracle.render.render over `walk`: (cls uint16, depth float32, index int32)"""
    flat = np.ascontiguousarray(cmap).reshape(-1)
    n = np.asarray(u).size
    cls = np.full(n, empty, np.uint16)
    depth = np.full(n, np.inf, np.float32)
    index = np.full(n, -1, np.int32)

    def visit(act, off, t):
        c = flat[off].astype(np.int64)
        hit = (c != empty) & (c != ignore)
        cls[act[hit]] = c[hit]
        depth[act[hit]] = t[hit].astype(np.float32)
        index[act[hit]] = off[hit]
        return hit

    walk(G, s, origin, voxel, cam, u, v, visit, near, far)
    return cls, depth, index


def render_probs(probs, G, s, origin, voxel, cam, u, v, class_map=None, empty=0, ignore=255, near=0.0, far=np.inf,
                 t_min=1e-4, lut=None):
    """(cls uint16, depth float32, opacity float32, probs float16 [n, C]) of pixels (u, v) of camera `cam` through
    one item's float16 probabilities `probs` [C, ...] (each plane read flat at i*s_x + j*s_y + k*s_z) and optional
    uint16 `class_map` (same layout; voxels holding `ignore` are skipped)"""
    P = np.ascontiguousarray(probs, np.float16)
    C = P.shape[0]
    P = P.reshape(C, -1)
    cm = None if class_map is None else np.ascontiguousarray(class_map).reshape(-1)
    n = np.asarray(u).size
    f32 = np.float32
    tm = f32(t_min)
    S = np.zeros((C, n), f32)
    T = np.ones(n, f32)
    D = np.full(n, -0.0, f32)                 # -0: addition's identity, as the kernel starts
    others = [c for c in range(C) if c != empty]

    def visit(act, off, t):
        keep = np.ones(act.size, bool)
        if cm is not None:
            keep &= cm[off].astype(np.int64) != ignore
        e = np.where(keep, P[empty, off].astype(f32), f32(1))
        keep &= e != f32(1)
        a, o, e, tau = act[keep], off[keep], e[keep], t[keep].astype(f32)
        Ta = T[a]
        for c in others:
            S[c, a] = S[c, a] + Ta * P[c, o].astype(f32)
        Tn = Ta * e
        D[a] = D[a] + (Ta - Tn) * tau
        T[a] = Tn
        stop = np.zeros(act.size, bool)
        stop[keep] = Tn <= tm
        return stop

    with np.errstate(invalid="ignore", over="ignore"):
        walk(G, s, origin, voxel, cam, u, v, visit, near, far)
        opacity = f32(1) - T
        depth = np.where(opacity > 0, D / np.where(opacity > 0, opacity, f32(1)), f32(np.inf)).astype(f32)
    ch = S.copy()
    ch[empty] = T
    best = ch[0].copy()
    cls = np.zeros(n, np.int64)
    for c in range(1, C):
        m = ch[c] > best
        best = np.where(m, ch[c], best)
        cls[m] = c
    if lut is not None:
        cls = np.asarray(lut, np.int64)[cls]
    return cls.astype(np.uint16), depth, opacity.astype(f32), ch.T.astype(np.float16)


def render_probs_image(probs, G, s, origin, voxel, cam, W, H, rows=None, **kw):
    """`render_probs` over rows `rows` (default every row) of a W x H view: cls, depth, opacity [len(rows), W] and
    probs [C, len(rows), W]"""
    rows = np.arange(H) if rows is None else np.asarray(rows)
    vv, uu = np.meshgrid(rows, np.arange(W), indexing="ij")
    cls, depth, opacity, p = render_probs(probs, G, s, origin, voxel, cam, uu.reshape(-1), vv.reshape(-1), **kw)
    shp = (len(rows), W)
    return cls.reshape(shp), depth.reshape(shp), opacity.reshape(shp), p.T.reshape((-1,) + shp)
