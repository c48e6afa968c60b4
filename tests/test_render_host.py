"""Camera views without a device: the kernel's ray walk (csrc/render.cuh, run on the CPU by
tests/host_emul/render_emul.cu) against the float64 numpy restatement (oracle/render.py) bit for bit, the oracle
against brute force and against the reference's voxel -> pixel projection, and the refusals of occd_render_classes,
render_classes, SceneMap.render and OccDepth.predict_view."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, fusion, render
from oracle import projection
from oracle import render as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("render_emul") / "librender_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "render_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).render_emulate
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_int,
                   C.c_double, C.c_double, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def run_emul(fn, cmap, G, s, origin, voxel, cam, u, v, empty=0, ignore=255, near=0.0, far=np.inf):
    m = np.ascontiguousarray(cmap, np.uint16).reshape(-1)
    Ga, sa = np.array(G, np.int32), np.array(s, np.int64)
    o, c = np.ascontiguousarray(origin, np.float64), np.ascontiguousarray(cam, np.float64)
    u, v = np.ascontiguousarray(u, np.int32).reshape(-1), np.ascontiguousarray(v, np.int32).reshape(-1)
    n = u.size
    cls, depth, index = np.full(n, 7, np.uint16), np.full(n, np.nan, np.float32), np.full(n, -7, np.int32)
    assert fn(m.ctypes.data, Ga.ctypes.data, sa.ctypes.data, o.ctypes.data, float(voxel), c.ctypes.data, empty, ignore,
              float(near), float(far), n, u.ctypes.data, v.ctypes.data, cls.ctypes.data, depth.ctypes.data,
              index.ctypes.data) == 0
    return cls, depth, index


def pixels(W, H):
    v, u = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return u.reshape(-1), v.reshape(-1)


def look(eye, yaw, pitch=0.0, roll=0.0):
    """E (grid -> camera) of a camera at `eye` whose optical axis (camera z) is grid +x turned by yaw about z and
    pitched down by `pitch`; camera x to the right, y down"""
    cz, sz, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
    fwd = np.array([cz * cp, sz * cp, -sp])
    right = np.array([sz, -cz, 0.0])
    down = np.cross(fwd, right)
    Rc = np.stack([right, down, fwd])          # rows: camera axes in the grid frame
    cr, sr = np.cos(roll), np.sin(roll)
    Rc = np.array([[cr, -sr, 0], [sr, cr, 0], [0, 0, 1]]) @ Rc
    E = np.eye(4)
    E[:3, :3] = Rc
    E[:3, 3] = -Rc @ np.asarray(eye, np.float64)
    return E


def intrinsics(f, W, H):
    return np.array([[f, 0.0, W / 2.0 - 0.3], [0.0, f * 1.01, H / 2.0 + 0.2], [0.0, 0.0, 1.0]])


def random_map(storage, density, seed, classes=20):
    g = np.random.default_rng(seed)
    m = g.integers(1, classes, size=storage).astype(np.uint16)
    m[g.random(storage) >= density] = 0
    m[g.random(storage) < 0.02] = 255
    return m


def check_bits(emul, cmap, G, s, origin, voxel, cam, u, v, **kw):
    got = run_emul(emul, cmap, G, s, origin, voxel, cam, u, v, **kw)
    want = ref.render(cmap, G, s, origin, voxel, cam, u, v, **kw)
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    return want


# ---- the host build of the kernel's walk against the oracle, bit for bit -------------------------------------------
def _cases():
    out = []
    rng = np.random.default_rng(11)
    for i in range(6):
        storage = tuple(int(x) for x in rng.integers(6, 20, 3))
        axes = "xyz" if i % 2 == 0 else "xzy"
        G, _ = ref.plane_layout(storage, axes)
        voxel = float(rng.uniform(0.1, 0.4))
        origin = tuple(rng.uniform(-2, 2, 3))
        ext = np.asarray(G) * voxel
        # outside, looking at the grid centre from a random side, or inside it
        centre = np.asarray(origin) + ext / 2
        if i < 4:
            yaw = rng.uniform(-np.pi, np.pi)
            eye = centre - 1.6 * np.linalg.norm(ext) * np.array([np.cos(yaw), np.sin(yaw), -0.3])
            E = look(eye, yaw, pitch=0.3, roll=rng.uniform(-0.2, 0.2))
        else:
            E = look(centre + rng.uniform(-0.2, 0.2, 3) * ext, rng.uniform(-np.pi, np.pi), rng.uniform(-0.5, 0.5))
        out.append(("random%d_%s" % (i, axes), storage, axes, origin, voxel, E, float(rng.uniform(0.05, 0.3))))
    return out


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_walk_matches_the_oracle_bit_for_bit(emul, case):
    _, storage, axes, origin, voxel, E, density = case
    W, H = 64, 48
    cmap = random_map(storage, density, 3)
    G, s = ref.plane_layout(storage, axes)
    cam = render.cameras(E, intrinsics(40.0, W, H))[0, 0]
    u, v = pixels(W, H)
    cls, depth, index = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v)
    hit = index >= 0
    assert 0 < int(hit.sum()) < hit.size or case[0].startswith("random4") or case[0].startswith("random5")
    assert hit.any()
    assert np.array_equal(cls[hit], cmap.reshape(-1)[index[hit]])
    assert ((cls[hit] != 0) & (cls[hit] != 255)).all() and (cls[~hit] == 0).all()
    assert np.isinf(depth[~hit]).all() and (depth[hit] >= 0).all()
    # near / far clip the same rays, in both builds
    dh = depth[hit]
    near = max(float(np.quantile(dh, 0.3)), 1.5 * voxel)            # the camera may sit in an occupied voxel
    far = max(float(np.quantile(dh, 0.8)), near + 2 * voxel)
    c2, d2, i2 = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v, near=near, far=far)
    h2 = i2 >= 0
    assert (d2[h2] >= np.float32(near)).all() and (d2[h2] <= np.float32(far)).all()
    assert h2.any() and not np.array_equal(i2, index)
    # another empty / ignore pair
    check_bits(emul, cmap, G, s, origin, voxel, cam, u, v, empty=255, ignore=0)


def _axis_camera(eye, f=4.0, c=(16, 12)):
    """E = identity rotation (camera axes = grid axes), K with a power-of-two focal length and integer centre: the
    column u = cx has d_x == 0 and the row v = cy has d_y == 0 exactly"""
    E = np.eye(4)
    E[:3, 3] = -np.asarray(eye, np.float64)
    K = np.array([[f, 0.0, c[0]], [0.0, f, c[1]], [0.0, 0.0, 1.0]])
    return E, K


def test_axis_parallel_rays_and_exact_edge_crossings(emul):
    """voxel 0.5 and a camera on lattice points: every value is exact in binary, the rays along the image diagonals
    cross x and y boundaries at the same time (edges; corners where z crosses too), and the centre row and column
    have d_a == 0"""
    storage, axes = (16, 16, 16), "xyz"
    G, s = ref.plane_layout(storage, axes)
    origin, voxel = (-4.0, -4.0, 0.0), 0.5
    W, H = 33, 25
    u, v = pixels(W, H)
    for eye in [(0.0, 0.0, -1.0), (-1.5, 0.5, -2.0), (0.0, 0.0, 1.0)]:       # the last inside the grid
        E, K = _axis_camera(eye)
        cam = render.cameras(E, K)[0, 0]
        d = (cam[0] * u + cam[1] * v) + cam[2], (cam[3] * u + cam[4] * v) + cam[5]
        assert (d[0] == 0).sum() == H and (d[1] == 0).sum() == W
        assert (np.abs(d[0]) == np.abs(d[1])).sum() > 40                   # edge crossings on the diagonals
        for density in (0.02, 0.1, 0.3):
            cmap = random_map(storage, density, int(density * 100))
            cls, depth, index = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v)
            assert (index >= 0).any()
    # the tie rule itself.  Pixel (20, 16): d = (1, 1, 1) from (0, 0, -1) enters the grid at t = 1 in voxel
    # (10, 10, 0) and crosses x, y and z boundaries together (a corner) every 0.5: x first, then y, then z, so the
    # corner at t = 2 leads from (11, 11, 1) to (12, 11, 1); y first would reach (11, 12, 1), z first (11, 11, 2)
    E, K = _axis_camera((0.0, 0.0, -1.0))
    cam = render.cameras(E, K)[0, 0]
    cmap = np.zeros(storage, np.uint16)
    cmap[12, 11, 1], cmap[11, 12, 1], cmap[11, 11, 2] = 3, 4, 6
    c, dd, ix = check_bits(emul, cmap, G, s, origin, voxel, cam, [20], [16])
    assert c[0] == 3 and ix[0] == 12 * s[0] + 11 * s[1] + 1 * s[2] and dd[0] == np.float32(2.0)
    cmap[12, 11, 1] = 0                                   # then (12, 12, 1) and (12, 12, 2), then the next corner
    cmap[12, 12, 2] = 9
    c, dd, ix = check_bits(emul, cmap, G, s, origin, voxel, cam, [20], [16])
    assert c[0] == 9 and dd[0] == np.float32(2.0)


def test_camera_inside_an_occupied_voxel(emul):
    storage = (10, 12, 8)
    G, s = ref.plane_layout(storage, "xyz")
    origin, voxel = (0.0, 0.0, 0.0), 0.25
    cmap = random_map(storage, 0.1, 5)
    eye = (1.3, 1.1, 0.9)
    i, j, k = (int(np.floor(e / voxel)) for e in eye)
    cmap[i, j, k] = 7
    W, H = 40, 30
    u, v = pixels(W, H)
    for yaw in (0.0, 1.0, 2.5):
        cam = render.cameras(look(eye, yaw, 0.4), intrinsics(30.0, W, H))[0, 0]
        cls, depth, index = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v)
        assert (cls == 7).all() and (index == i * s[0] + j * s[1] + k * s[2]).all() and (depth == 0).all()
        # past the voxel with near: the rays go on through the grid
        cls, depth, index = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v, near=0.5)
        assert (depth[index >= 0] >= 0.5).all() and not (cls == 7).all()


def test_grid_behind_the_camera_and_empty_map(emul):
    storage = (12, 12, 6)
    G, s = ref.plane_layout(storage, "xyz")
    origin, voxel = (0.0, 0.0, 0.0), 0.2
    W, H = 48, 32
    u, v = pixels(W, H)
    cmap = random_map(storage, 0.5, 9)
    cam = render.cameras(look((-1.0, 1.2, 0.6), np.pi), intrinsics(30.0, W, H))[0, 0]     # looking away
    cls, depth, index = check_bits(emul, cmap, G, s, origin, voxel, cam, u, v)
    assert (index == -1).all() and np.isinf(depth).all() and (cls == 0).all()
    cam = render.cameras(look((-1.0, 1.2, 0.6), 0.0), intrinsics(30.0, W, H))[0, 0]      # looking at it
    assert (check_bits(emul, cmap, G, s, origin, voxel, cam, u, v)[2] >= 0).any()
    empty = np.zeros(storage, np.uint16)
    empty[::2] = 255                                                                     # ignore is transparent too
    cls, depth, index = check_bits(emul, empty, G, s, origin, voxel, cam, u, v)
    assert (index == -1).all() and np.isinf(depth).all() and (cls == 0).all()


# ---- the oracle against independent code ----------------------------------------------------------------------------
def _slab(o, d, lo, hi):
    """entry and exit times of the ray o + t d through the box [lo, hi) (float64, the textbook slab test)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (lo - o) / d, (hi - o) / d
    tmin, tmax = np.minimum(t1, t2), np.maximum(t1, t2)
    par = d == 0
    inside = (o >= lo) & (o < hi)
    tmin = np.where(par, np.where(inside, -np.inf, np.inf), tmin)
    tmax = np.where(par, np.where(inside, np.inf, -np.inf), tmax)
    return tmin.max(-1), tmax.min(-1)


@pytest.mark.parametrize("seed", range(4))
def test_oracle_against_brute_force(seed):
    """away from ties, the hit is the occupied voxel with the least entry time among those the ray meets inside
    [near, far]; a miss meets none"""
    rng = np.random.default_rng(200 + seed)
    storage = tuple(int(x) for x in rng.integers(4, 9, 3))
    axes = "xyz" if seed % 2 == 0 else "xzy"
    G, s = ref.plane_layout(storage, axes)
    voxel = float(rng.uniform(0.2, 0.5))
    origin = rng.uniform(-1, 1, 3)
    cmap = random_map(storage, 0.12, seed)
    W, H = 40, 30
    u, v = pixels(W, H)
    centre = origin + np.asarray(G) * voxel / 2
    eye = centre + rng.uniform(-1, 1, 3) * np.asarray(G) * voxel * (0.3 if seed == 3 else 1.2)
    to = centre - eye + rng.uniform(-0.2, 0.2, 3) * voxel
    yaw, pitch = np.arctan2(to[1], to[0]), np.arctan2(-to[2], np.hypot(to[0], to[1]))   # looking at the centre
    cam = render.cameras(look(eye, yaw, pitch), intrinsics(25.0, W, H))[0, 0]
    near, far = (0.0, np.inf) if seed < 2 else (0.3, 2.0)
    cls, depth, index = ref.render(cmap, G, s, origin, voxel, cam, u, v, near=near, far=far)
    # every occupied voxel's box, in storage order
    occ = np.argwhere((cmap != 0) & (cmap != 255))
    ijk = occ[:, [0, 2, 1]] if axes == "xzy" else occ
    lo = origin + ijk * voxel
    off = (ijk * np.asarray(s)).sum(1)
    M, o = cam[:9].reshape(3, 3), cam[9:]
    d = np.stack([u, v, np.ones_like(u)], 1).astype(np.float64) @ M.T
    checked = 0
    for p in range(u.size):
        tin, tout = _slab(o, d[p], lo, lo + voxel)
        a, b = np.maximum(tin, near), np.minimum(tout, far)
        margin = b - a
        if (np.abs(margin) < 1e-9).any():
            continue                                       # grazes a voxel edge: a tie
        meet = margin > 0
        if not meet.any():
            assert index[p] == -1 and np.isinf(depth[p]), p
            checked += 1
            continue
        order = np.sort(a[meet])
        if order.size > 1 and order[1] - order[0] < 1e-9:
            continue                                       # two voxels entered at the same time
        best = np.flatnonzero(meet)[np.argmin(a[meet])]
        assert index[p] == off[best], (p, index[p], off[best])
        assert abs(float(depth[p]) - a[best]) <= 1e-6 * max(1.0, a[best]), (p, depth[p], a[best])
        checked += 1
    assert checked > 0.95 * u.size and (index >= 0).sum() > 50


def _projection_check(E, K, vox_origin, voxel, scene_size, W, H, axes, n, seed):
    """one-voxel maps: the pixel vox2pix projects the voxel's centre to renders that voxel"""
    pix, fov, z = projection.vox2pix(E, K, vox_origin, voxel, W, H, scene_size, 0)
    dims = np.ceil(np.asarray(scene_size) / voxel).astype(int)           # x, y, z
    storage = tuple(dims) if axes == "xyz" else (dims[0], dims[2], dims[1])
    G, s = ref.plane_layout(storage, axes)
    cam = ref.camera(E, K)
    inside = np.flatnonzero(fov[:, 0])
    pick = np.random.default_rng(seed).choice(inside, n, replace=False)
    for q in pick:
        x, y, zz = np.unravel_index(q, tuple(dims))
        cmap = np.zeros(storage, np.uint16)
        off = x * s[0] + y * s[1] + zz * s[2]
        cmap.reshape(-1)[off] = 5
        c, d, i = ref.render(cmap, G, s, vox_origin, voxel, cam, [pix[q, 0, 0]], [pix[q, 0, 1]])
        assert i[0] == off and c[0] == 5, (q, x, y, zz, pix[q, 0])
        assert abs(float(d[0]) - z[q]) < voxel, (d[0], z[q])


def test_oracle_against_the_reference_projection_kitti():
    sys.path.insert(0, ROOT)
    import synthetic
    W, H = 1220, 370
    K, Ts = synthetic.kitti_calib(W, H)
    for v in range(2):
        _projection_check(np.asarray(Ts[v], np.float64), K, np.array([0.0, -25.6, -2.0]), 0.2, (51.2, 51.2, 6.4),
                          W, H, "xyz", 12, v)


def test_oracle_against_the_reference_projection_nyu():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from camera_frames import nyu_frame, NYU_K
    f = nyu_frame(1, with_depth=False)
    E = np.linalg.inv(f["cam_pose"])
    _projection_check(E, NYU_K, f["vox_origin"], 0.08, (4.8, 4.8, 2.88), 640, 480, "xzy", 12, 3)


# ---- refusals of the entry point, without a device ------------------------------------------------------------------
def _lib_built():
    _build.build()
    return _lib.lib()


def _render_args(**k):
    buf = np.zeros(64, np.uint16)
    p = buf.ctypes.data
    a = dict(map=p, B=1, GX=4, GY=4, GZ=2, strides=np.array([8, 2, 1], np.int64), origin=np.zeros(3), voxel=0.2,
             V=1, cams=np.tile(np.r_[np.eye(3).reshape(-1), 0.0, 0.0, -1.0], 1), W=8, H=4, empty=0, ignore=255,
             near=0.0, far=np.inf, cls=p, depth=None, index=None)
    a.update(k)
    keep = [buf] + [v for v in a.values() if isinstance(v, np.ndarray)]
    ptr = lambda v: v.ctypes.data if isinstance(v, np.ndarray) else v      # noqa: E731
    args = (a["map"], a["B"], a["GX"], a["GY"], a["GZ"], ptr(a["strides"]), ptr(a["origin"]), a["voxel"], a["V"],
            ptr(a["cams"]), a["W"], a["H"], a["empty"], a["ignore"], a["near"], a["far"], ptr(a["cls"]),
            ptr(a["depth"]), ptr(a["index"]), None)
    return args, keep


RENDER_BAD = {
    "map": dict(map=None), "strides_null": dict(strides=None), "origin_null": dict(origin=None),
    "cams_null": dict(cams=None), "no_output": dict(cls=None), "B0": dict(B=0), "V0": dict(V=0),
    "cameras33": dict(B=3, V=11), "GX": dict(GX=0), "GZ": dict(GZ=-2), "voxels": dict(GX=2048, GY=2048, GZ=512),
    "stride_neg": dict(strides=np.array([8, -2, 1], np.int64)),
    "stride_out": dict(strides=np.array([16, 2, 1], np.int64)), "W0": dict(W=0), "H0": dict(H=0),
    "H_big": dict(H=70000), "voxel0": dict(voxel=0.0), "voxel_nan": dict(voxel=float("nan")),
    "origin_inf": dict(origin=np.array([0.0, np.inf, 0.0])), "cams_nan": dict(cams=np.full(12, np.nan)),
    "empty": dict(empty=-1), "ignore": dict(ignore=65536), "near_neg": dict(near=-0.1),
    "near_inf": dict(near=np.inf), "far": dict(near=1.0, far=1.0), "far_nan": dict(far=float("nan")),
    "align": dict(depth=np.zeros(8, np.uint8).ctypes.data + 1),
}


@pytest.mark.parametrize("case", sorted(RENDER_BAD))
def test_render_refusals(case):
    L = _lib_built()
    args, keep = _render_args(**RENDER_BAD[case])
    assert L.occd_render_classes(*args) == _lib.ERR_ARG, case
    assert L.occd_last_error().startswith(b"occd_render_classes: "), L.occd_last_error()


# ---- render_classes, SceneMap.render, predict_view: host-side refusals -------------------------------------------
def _K():
    return np.array([[100.0, 0, 32], [0, 100.0, 24], [0, 0, 1]])


def test_render_classes_refusals(monkeypatch):
    called = []
    monkeypatch.setattr(_lib, "lib", lambda: called.append(1))
    m = torch.zeros(2, 8, 6, 4, dtype=torch.uint16)
    E, K = np.eye(4), _K()
    go = lambda **kw: render.render_classes(**dict(dict(class_map=m, E=E, K=K, size=(64, 48),   # noqa: E731
                                                        grid_origin=(0, 0, 0), grid_voxel=0.2), **kw))
    with pytest.raises(TypeError, match="uint16"):
        go(class_map=m.int())
    with pytest.raises(ValueError, match="contiguous"):
        go(class_map=m.transpose(1, 2))
    with pytest.raises(ValueError, match="contiguous"):
        go(class_map=m[0, 0])
    with pytest.raises(ValueError, match="axes"):
        go(axes="zyx")
    for size in [(0, 48), (64, -1), (64,), "ab", (64, 70000)]:
        with pytest.raises(ValueError, match="size"):
            go(size=size)
    with pytest.raises(ValueError, match="grid_origin"):
        go(grid_origin=(0, 0))
    with pytest.raises(ValueError, match="grid_voxel"):
        go(grid_voxel=0.0)
    with pytest.raises(ValueError, match="empty and ignore"):
        go(ignore=70000)
    for near, far in [(-1.0, 10.0), (2.0, 2.0), (np.nan, 1.0), (0.0, np.nan), (np.inf, np.inf)]:
        with pytest.raises(ValueError, match="near"):
            go(near=near, far=far)
    for bad in [np.full((4, 4), np.nan), np.zeros((4, 4)), np.eye(3)]:
        with pytest.raises(ValueError, match="render_classes: E"):
            go(E=bad)
    with pytest.raises(ValueError, match="E holds 3 items"):
        go(E=np.stack([np.eye(4)] * 3))
    with pytest.raises(ValueError, match="last row"):
        go(K=np.array([[100.0, 0, 32], [0, 100, 24], [0, 0, 2]]))
    with pytest.raises(ValueError, match="singular"):
        go(K=np.array([[0.0, 0, 32], [0, 100, 24], [0, 0, 1]]))
    with pytest.raises(ValueError, match="K must be finite"):
        go(K=np.array([[np.inf, 0, 32], [0, 100, 24], [0, 0, 1]]))
    with pytest.raises(ValueError, match="E holds 2 cameras per item, K 3"):
        go(E=np.stack([np.stack([np.eye(4)] * 2)] * 2), K=np.stack([np.stack([_K()] * 3)] * 2))
    with pytest.raises(ValueError, match="at most 32 cameras"):
        go(E=np.stack([np.stack([np.eye(4)] * 17)] * 2))
    shape = (2, 1, 48, 64)
    outs = [torch.empty(shape, dtype=torch.uint16), torch.empty(shape), torch.empty(shape, dtype=torch.int32)]
    with pytest.raises(ValueError, match="at least one"):
        go(out=render.View(None, None, None))
    with pytest.raises(TypeError, match="out.depth"):
        go(out=render.View(outs[0], outs[2], None))
    with pytest.raises(ValueError, match="out.index"):
        go(out=render.View(None, None, outs[2][:, :, :, :32]))
    with pytest.raises(ValueError, match="out.classes"):
        go(out=render.View(torch.empty(2, 2, 48, 64, dtype=torch.uint16), None, None))
    # every argument good: the class map on the CPU is the last refusal before the launch
    with pytest.raises(ValueError, match="CUDA device"):
        go(out=render.View(*outs))
    with pytest.raises(ValueError, match="CUDA device"):
        go(E=np.stack([np.stack([np.eye(4)] * 16)] * 2), near=0.5, far=80.0)
    assert not called


def test_cameras_follow_the_header():
    """M = R^-1 K^-1 and o = -R^-1 t: o is the camera centre, and M (u, v, 1) is the ray whose camera z grows by 1
    per unit of t"""
    E = look((1.0, -2.0, 0.5), 0.7, 0.2, 0.1)
    K = intrinsics(500.0, 640, 480)
    cams = render.cameras(np.stack([E, E]), K, B=2)
    assert cams.shape == (2, 1, 12) and np.array_equal(cams[0], cams[1])
    assert np.array_equal(cams[0, 0], ref.camera(E, K))
    M, o = cams[0, 0, :9].reshape(3, 3), cams[0, 0, 9:]
    assert np.allclose(o, [1.0, -2.0, 0.5])
    p = o + 3.0 * (M @ np.array([100.0, 50.0, 1.0]))
    q = E @ np.append(p, 1.0)
    assert np.isclose(q[2], 3.0) and np.allclose(K @ (q[:3] / q[2]), [100.0, 50.0, 1.0])


def _cpu_map(C=4, dims=(4, 4, 2)):
    m = object.__new__(fusion.SceneMap)
    m.n_classes, m.dims, m.voxel, m.min_prob = C, dims, 0.2, 1e-3
    m.origin, m.device = np.zeros(3), torch.device("cpu")
    m._acc = torch.zeros((C,) + dims)
    m._count = torch.zeros(dims, dtype=torch.int32)
    m._spare = None
    return m


def test_scene_map_render_refuses_before_any_launch(monkeypatch):
    called = []
    monkeypatch.setattr(_lib, "lib", lambda: called.append(1))
    monkeypatch.setattr(fusion.SceneMap, "classes", lambda *a, **k: called.append(2))
    m = _cpu_map()
    K = _K()
    with pytest.raises(ValueError, match="SceneMap.render: unknown"):
        m.render(np.eye(4), K, (64, 48), unknown=-1)
    with pytest.raises(ValueError, match="SceneMap.render: E"):
        m.render(np.full((4, 4), np.nan), K, (64, 48))
    with pytest.raises(ValueError, match="SceneMap.render: K's last row"):
        m.render(np.eye(4), np.eye(3) * 2, (64, 48))
    with pytest.raises(ValueError, match="SceneMap.render: size"):
        m.render(np.eye(4), K, (0, 48))
    with pytest.raises(ValueError, match="SceneMap.render: near"):
        m.render(np.eye(4), K, (64, 48), near=3.0, far=1.0)
    with pytest.raises(ValueError, match="SceneMap.render: E holds 2 items"):
        m.render(np.stack([np.eye(4)] * 2), K, (64, 48))
    with pytest.raises(ValueError, match="at most 32"):
        m.render(np.stack([np.eye(4)] * 33)[None], K, (64, 48))
    assert not called


@pytest.fixture(scope="module")
def kitti_model():
    if os.path.join(ROOT, "tools") not in sys.path:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
    import shipped_configs
    m, _, _ = shipped_configs.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=(96, 320), full=(64, 64, 16))
    return m


def _kitti(V=2, H=96, W=320, T=None, K=None):
    return {"img": np.zeros((V, H, W, 3), np.uint8), "cam_k": np.stack([np.eye(3)] * V) if K is None else K,
            "T_velo_2_cam": np.stack([np.eye(4)] * V) if T is None else T, "img_hw": (H, W),
            "scene_size": (12.8, 12.8, 3.2), "vox_origin": np.array([0.0, -6.4, -2.0]), "voxel_size": 0.4}


def test_predict_view_refusals(kitti_model, monkeypatch):
    m = kitti_model
    ran = []
    monkeypatch.setattr(m, "_run_frames", lambda *a, **k: ran.append(1))
    monkeypatch.setattr(m, "_run_frame", lambda *a, **k: ran.append(1))
    monkeypatch.setattr(m, "_check_mode", lambda x: None)          # the frames' host side runs without a device
    with pytest.raises(ValueError, match="views"):
        m.predict_view(_kitti(), views=(0.5,))
    with pytest.raises(ValueError, match="1 to 32 cameras"):
        m.predict_view(_kitti(), views=())
    with pytest.raises(ValueError, match="1 to 32 cameras"):
        m.predict_view([_kitti()] * 17, views=(0, 1))
    with pytest.raises(ValueError, match="views \\(0, 2\\) of a frame with 2 cameras"):
        m.predict_view(_kitti(), views=(0, 2))
    with pytest.raises(ValueError, match="views \\(-1,\\)"):
        m.predict_view([_kitti(), _kitti()], views=(-1,))
    with pytest.raises(ValueError, match="predict_view: near"):
        m.predict_view(_kitti(), near=-1.0)
    with pytest.raises(ValueError, match="predict_view: near"):
        m.predict_view(_kitti(), near=5.0, far=5.0)
    bad_T = np.stack([np.eye(4), np.zeros((4, 4))])
    with pytest.raises(ValueError, match="predict_view: E is singular"):
        m.predict_view(_kitti(T=bad_T), views=(0, 1))
    m.predict_view(_kitti(T=bad_T), views=(0,))                        # view 1 not asked for
    bad_K = np.stack([np.eye(3), np.diag([1.0, 1.0, 2.0])])
    with pytest.raises(ValueError, match="predict_view: K's last row"):
        m.predict_view([_kitti(), _kitti(K=bad_K)], views=(1,))
    with pytest.raises(TypeError, match="frame dict or a list"):
        m.predict_view(object())
    assert len(ran) == 1
    from occdepth_b200.parallel import SimSlabGroup
    m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
    try:
        with pytest.raises(NotImplementedError, match="slab"):
            m.predict_view(_kitti())
    finally:
        m.__dict__.pop("slab_ctx", None)
    assert len(ran) == 1
