"""Soft camera views without a device: the kernel's compositing (csrc/render.cuh, run on the CPU by
tests/host_emul/render_probs_emul.cu) against the numpy restatement (oracle/render_probs.py) bit for bit, the soft
render of one-hot fields against the hard render, the oracle against a float64 brute-force compositor, the ptxas logs
of the render kernels, and the refusals of occd_render_probs, render_probs, SceneMap.render_probs and
OccDepth.predict_view(soft=True)."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, render
from oracle import render as ref_hard
from oracle import render_probs as ref

from test_render_host import (_axis_camera, _cpu_map, _K, _kitti, _slab, emul, intrinsics, kitti_model,  # noqa: F401
                              look, pixels, random_map, run_emul)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASS_COUNTS = (3, 12, 16, 17, 20, 33, 64)          # every instantiation (16, 32, 64) and both sides of each boundary


@pytest.fixture(scope="module")
def soft(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("render_probs_emul") / "librender_probs_emul.so"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "--expt-relaxed-constexpr",
           "-shared", "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "occdepth_b200", "csrc"),
           "-o", str(out), os.path.join(ROOT, "tests", "host_emul", "render_probs_emul.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    fn = C.CDLL(str(out)).render_probs_emulate
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                   C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_float, C.c_void_p, C.c_longlong,
                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


def run_soft(fn, probs, G, s, origin, voxel, cam, u, v, class_map=None, empty=0, ignore=255, near=0.0, far=np.inf,
             t_min=1e-4, lut=None):
    P = np.ascontiguousarray(probs, np.float16)
    Cn = P.shape[0]
    cm = None if class_map is None else np.ascontiguousarray(class_map, np.uint16).reshape(-1)
    lt = None if lut is None else np.ascontiguousarray(np.asarray(lut).astype(np.int64).astype(np.uint16))
    Ga, sa = np.array(G, np.int32), np.array(s, np.int64)
    o, c = np.ascontiguousarray(origin, np.float64), np.ascontiguousarray(cam, np.float64)
    u, v = np.ascontiguousarray(u, np.int32).reshape(-1), np.ascontiguousarray(v, np.int32).reshape(-1)
    n = u.size
    cls, depth = np.full(n, 7, np.uint16), np.full(n, np.nan, np.float32)
    opa, po = np.full(n, np.nan, np.float32), np.full((n, Cn), np.nan, np.float16)
    ptr = lambda x: None if x is None else x.ctypes.data       # noqa: E731
    assert fn(P.ctypes.data, Cn, P[0].size, ptr(cm), Ga.ctypes.data, sa.ctypes.data, o.ctypes.data, float(voxel),
              c.ctypes.data, empty, ignore, float(near), float(far), float(t_min), ptr(lt), n, u.ctypes.data,
              v.ctypes.data, cls.ctypes.data, depth.ctypes.data, opa.ctypes.data, po.ctypes.data) == 0
    return cls, depth, opa, po


def canon(x):
    """x's bytes with every NaN one value: a NaN's sign and payload are not part of the arithmetic"""
    if x.dtype.kind == "f":
        x = np.where(np.isnan(x), x.dtype.type(np.nan), x)
    return x.tobytes()


def check_bits(fn, probs, G, s, origin, voxel, cam, u, v, **kw):
    got = run_soft(fn, probs, G, s, origin, voxel, cam, u, v, **kw)
    want = ref.render_probs(probs, G, s, origin, voxel, cam, u, v, **kw)
    for name, g, w in zip(("cls", "depth", "opacity", "probs"), got, want):
        assert canon(g) == canon(w), name
    return want


def soft_field(storage, Cn, seed, surface=0.15, free=0.6):
    """float16 [C, *storage], channel 0 empty: a fraction `free` of voxels certainly free (p(empty) == 1 exactly),
    a fraction `surface` confident surfaces, the rest soft (rays cross them partly), a few one-hot; class map the
    arg-max"""
    g = np.random.default_rng(seed)
    logits = g.normal(0.0, 1.5, (Cn,) + storage)
    kind = g.random(storage)
    logits[0] += np.where(kind < free, 0.0, np.where(kind < free + surface, -6.0, -1.0))
    p = np.exp(logits - logits.max(0))
    p /= p.sum(0)
    p = p.astype(np.float16)
    p[:, kind < free] = 0
    p[0, kind < free] = 1
    onehot = g.random(storage) < 0.03
    k = g.integers(1, Cn, storage) if Cn > 1 else np.zeros(storage, np.int64)
    for c in range(Cn):
        p[c][onehot] = np.float16(c == k[onehot])
    cmap = p.astype(np.float32).argmax(0).astype(np.uint16)
    cmap[g.random(storage) < 0.05] = 255
    return p, cmap


def _camera_case(i, storage, axes, rng):
    G, _ = ref.plane_layout(storage, axes)
    voxel = float(rng.uniform(0.1, 0.4))
    origin = tuple(rng.uniform(-2, 2, 3))
    ext = np.asarray(G) * voxel
    centre = np.asarray(origin) + ext / 2
    if i % 3 != 2:                                         # outside, looking at the grid
        yaw = rng.uniform(-np.pi, np.pi)
        eye = centre - 1.6 * np.linalg.norm(ext) * np.array([np.cos(yaw), np.sin(yaw), -0.3])
        E = look(eye, yaw, pitch=0.3, roll=rng.uniform(-0.2, 0.2))
    else:                                                  # inside it
        E = look(centre + rng.uniform(-0.2, 0.2, 3) * ext, rng.uniform(-np.pi, np.pi), rng.uniform(-0.5, 0.5))
    return G, origin, voxel, E


# ---- the host build of the compositing against the oracle, bit for bit ---------------------------------------------
@pytest.mark.parametrize("Cn", CLASS_COUNTS)
def test_compositing_matches_the_oracle_bit_for_bit(soft, Cn):
    rng = np.random.default_rng(100 + Cn)
    W, H = 40, 30
    u, v = pixels(W, H)
    for i in range(3):
        storage = tuple(int(x) for x in rng.integers(6, 16, 3))
        axes = "xyz" if i % 2 == 0 else "xzy"
        G, origin, voxel, E = _camera_case(i, storage, axes, rng)
        _, s = ref.plane_layout(storage, axes)
        probs, cmap = soft_field(storage, Cn, 7 * Cn + i)
        cam = render.cameras(E, intrinsics(30.0, W, H))[0, 0]
        lut = rng.integers(0, 300, Cn)
        cls, depth, opa, _ = check_bits(soft, probs, G, s, origin, voxel, cam, u, v)
        assert (opa > 0).any() and ((opa > 0) & (opa < 1)).any()
        check_bits(soft, probs, G, s, origin, voxel, cam, u, v, class_map=cmap, t_min=0.0, lut=lut)
        check_bits(soft, probs, G, s, origin, voxel, cam, u, v, class_map=cmap, ignore=int(cmap.reshape(-1)[0]),
                   t_min=0.05)
        hit = np.isfinite(depth)
        near = max(float(np.quantile(depth[hit], 0.3)), 1.5 * voxel) if hit.any() else 0.5
        far = near + 4 * voxel
        check_bits(soft, probs, G, s, origin, voxel, cam, u, v, near=near, far=far, t_min=0.0)
        if Cn > 2:                                          # another channel as empty
            check_bits(soft, probs, G, s, origin, voxel, cam, u, v, empty=Cn - 1, lut=lut)


def test_axis_parallel_rays_and_exact_edge_crossings(soft):
    storage, axes = (16, 16, 16), "xyz"
    G, s = ref.plane_layout(storage, axes)
    origin, voxel = (-4.0, -4.0, 0.0), 0.5
    W, H = 33, 25
    u, v = pixels(W, H)
    for eye in [(0.0, 0.0, -1.0), (-1.5, 0.5, -2.0), (0.0, 0.0, 1.0)]:
        E, K = _axis_camera(eye)
        cam = render.cameras(E, K)[0, 0]
        for Cn, seed in ((5, 1), (20, 2)):
            probs, cmap = soft_field(storage, Cn, seed, surface=0.05, free=0.85)
            check_bits(soft, probs, G, s, origin, voxel, cam, u, v)
            check_bits(soft, probs, G, s, origin, voxel, cam, u, v, class_map=cmap, t_min=0.0)


def test_nan_and_out_of_range_probabilities_are_not_touched(soft):
    storage, axes = (10, 8, 6), "xzy"
    G, s = ref.plane_layout(storage, axes)
    probs, _ = soft_field(storage, 6, 4, surface=0.1, free=0.4)
    g = np.random.default_rng(5)
    flat = probs.reshape(6, -1)
    flat[:, g.random(flat.shape[1]) < 0.05] = np.float16(np.nan)
    flat[2, g.random(flat.shape[1]) < 0.1] = np.float16(1.5)
    flat[0, g.random(flat.shape[1]) < 0.05] = np.float16(-0.25)
    W, H = 32, 24
    u, v = pixels(W, H)
    cam = render.cameras(look((-1.5, 0.3, 0.5), 0.1, 0.2), intrinsics(25.0, W, H))[0, 0]
    cls, depth, opa, p = check_bits(soft, probs, G, s, (0.0, 0.0, 0.0), 0.1, cam, u, v, t_min=0.0)
    assert np.isnan(opa).any() and np.isnan(p.astype(np.float32)).any()


# ---- one-hot fields: the soft render is the hard render ------------------------------------------------------------
@pytest.mark.parametrize("Cn", (20, 33))
def test_one_hot_fields_render_as_the_hard_render(soft, emul, Cn):
    rng = np.random.default_rng(Cn)
    W, H = 48, 36
    u, v = pixels(W, H)
    for i in range(3):
        storage = tuple(int(x) for x in rng.integers(8, 18, 3))
        axes = "xyz" if i % 2 == 0 else "xzy"
        G, origin, voxel, E = _camera_case(i, storage, axes, rng)
        _, s = ref.plane_layout(storage, axes)
        cmap = random_map(storage, 0.1, i, classes=Cn)     # classes 1..Cn-1, 0 empty, some 255 (ignore)
        probs = np.zeros((Cn,) + storage, np.float16)
        for c in range(Cn):
            probs[c][cmap == c] = 1
        probs[0][cmap == 255] = np.float16(0.5)              # what ignore hides must not matter
        probs[1][cmap == 255] = np.float16(0.5)
        cam = render.cameras(E, intrinsics(30.0, W, H))[0, 0]
        hd = run_emul(emul, cmap, G, s, origin, voxel, cam, u, v)[1]
        assert np.isfinite(hd).any() and np.isinf(hd).any()
        near = float(np.quantile(hd[np.isfinite(hd)], 0.5))
        for kw in (dict(), dict(near=near, far=near + 6 * voxel)):
            hc, hd, hi = run_emul(emul, cmap, G, s, origin, voxel, cam, u, v, **kw)
            for t_min in (0.0, 1e-4):
                sc, sd, so, sp = check_bits(soft, probs, G, s, origin, voxel, cam, u, v, class_map=cmap,
                                            t_min=t_min, **kw)
                assert sc.tobytes() == hc.tobytes() and sd.tobytes() == hd.tobytes()
                assert np.array_equal(so, (hi >= 0).astype(np.float32))


def test_one_hot_camera_on_a_voxel_boundary(soft, emul):
    """a camera exactly on a voxel boundary, inside an occupied voxel: the hard render's entry time is -0 there
    (max(+0, -0) keeps the later operand), and the soft depth keeps that sign because its sum starts at -0"""
    storage, axes, Cn = (40, 36, 12), "xyz", 20
    G, s = ref.plane_layout(storage, axes)
    cmap = random_map(storage, 0.08, 5, classes=Cn)
    probs = np.zeros((Cn,) + storage, np.float16)
    for c in range(Cn):
        probs[c][cmap == c] = 1
    origin, voxel = np.array([-1.0, -3.6, -1.2]), 0.2
    centre = origin + np.asarray(G) * voxel / 2
    W, H = 96, 64
    u, v = pixels(W, H)
    cam = render.cameras(look(centre + np.array([0.2, 0.3, 0.1]), 2.0, 0.1), intrinsics(80.0, W, H))[0, 0]
    hc, hd, hi = run_emul(emul, cmap, G, s, origin, voxel, cam, u, v)
    assert (np.signbit(hd) & (hd == 0)).any()
    sc, sd, so, _ = check_bits(soft, probs, G, s, origin, voxel, cam, u, v, class_map=cmap)
    assert sc.tobytes() == hc.tobytes() and sd.tobytes() == hd.tobytes()
    assert np.array_equal(so, (hi >= 0).astype(np.float32))


def test_oracle_walk_is_the_hard_walk():
    """the walk under render_probs gives oracle.render.render's hard view bit for bit"""
    rng = np.random.default_rng(3)
    W, H = 40, 30
    u, v = pixels(W, H)
    for i in range(4):
        storage = tuple(int(x) for x in rng.integers(6, 16, 3))
        axes = "xyz" if i % 2 == 0 else "xzy"
        G, origin, voxel, E = _camera_case(i, storage, axes, rng)
        _, s = ref.plane_layout(storage, axes)
        cmap = random_map(storage, 0.1, i)
        cam = render.cameras(E, intrinsics(30.0, W, H))[0, 0]
        for kw in (dict(), dict(near=0.5, far=2.0), dict(empty=255, ignore=0)):
            a = ref.render_hard(cmap, G, s, origin, voxel, cam, u, v, **kw)
            b = ref_hard.render(cmap, G, s, origin, voxel, cam, u, v, **kw)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


# ---- the oracle against a float64 brute-force compositor -----------------------------------------------------------
@pytest.mark.parametrize("seed", range(3))
def test_oracle_against_brute_force(seed):
    """away from ties: every voxel the ray meets in [near, far], by slab test, sorted by entry time and composited in
    float64 -- channels within float32 tolerance, their sum the composited input mass, depth between the first and last
    contributing entry, opacity 1 - T"""
    rng = np.random.default_rng(300 + seed)
    storage = tuple(int(x) for x in rng.integers(4, 9, 3))
    axes = "xyz" if seed % 2 == 0 else "xzy"
    G, s = ref.plane_layout(storage, axes)
    voxel = float(rng.uniform(0.2, 0.5))
    origin = rng.uniform(-1, 1, 3)
    Cn = (5, 17, 40)[seed]
    probs, _ = soft_field(storage, Cn, seed, surface=0.05, free=0.5)
    W, H = 32, 24
    u, v = pixels(W, H)
    centre = origin + np.asarray(G) * voxel / 2
    eye = centre + rng.uniform(-1, 1, 3) * np.asarray(G) * voxel * 1.2
    to = centre - eye
    cam = render.cameras(look(eye, np.arctan2(to[1], to[0]), np.arctan2(-to[2], np.hypot(to[0], to[1]))),
                         intrinsics(20.0, W, H))[0, 0]
    near, far = (0.0, np.inf) if seed < 2 else (0.3, 2.5)
    cls, depth, opa, p = ref.render_probs(probs, G, s, origin, voxel, cam, u, v, near=near, far=far, t_min=0.0)
    P = probs.reshape(Cn, -1).astype(np.float64)
    allv = np.argwhere(np.ones(storage, bool))
    ijk = allv[:, [0, 2, 1]] if axes == "xzy" else allv
    lo = origin + ijk * voxel
    off = (ijk * np.asarray(s)).sum(1)
    M, o = cam[:9].reshape(3, 3), cam[9:]
    d = np.stack([u, v, np.ones_like(u)], 1).astype(np.float64) @ M.T
    checked = 0
    for q in range(u.size):
        tin, tout = _slab(o, d[q], lo, lo + voxel)
        a, b = np.maximum(tin, near), np.minimum(tout, far)
        margin = b - a
        if (np.abs(margin) < 1e-9).any():
            continue                                       # grazes a voxel edge: a tie
        meet = np.flatnonzero(margin > 0)
        order = meet[np.argsort(a[meet], kind="stable")]
        if order.size > 1 and np.min(np.diff(a[order])) < 1e-9:
            continue
        T, S, D, mass, ts = 1.0, np.zeros(Cn), 0.0, 0.0, []
        for k in order:
            pk = P[:, off[k]]
            if pk[0] == 1.0:
                continue
            S[1:] += T * pk[1:]
            mass += T * (pk.sum() - pk[0])
            D += T * (1 - pk[0]) * a[k]
            ts.append(a[k])
            T *= pk[0]
        got = p[q].astype(np.float64)
        assert abs(float(opa[q]) - (1 - T)) <= 1e-5, q
        assert np.allclose(got[1:], S[1:], atol=2e-3, rtol=2e-3), q        # float16 outputs
        assert abs(got[0] - T) <= 2e-3, q
        assert abs(float(p[q].astype(np.float32).sum(dtype=np.float64)) - (T + mass)) <= 2e-3 * Cn, q
        if ts and 1 - T > 1e-6:
            assert min(ts) * (1 - 1e-5) - 1e-6 <= depth[q] <= max(ts) * (1 + 1e-5) + 1e-6, q
            assert abs(float(depth[q]) - D / (1 - T)) <= 1e-4 * max(1.0, max(ts)), q
        else:
            assert np.isinf(depth[q]) or 1 - T <= 1e-6
        checked += 1
    assert checked > 0.9 * u.size and (opa > 0.5).sum() > 20


# ---- the ptxas logs of the render kernels ---------------------------------------------------------------------------
def test_render_kernels_neither_spill_nor_use_a_stack():
    _build.build()
    log = open(os.path.join(_build.OBJDIR, "render.o.log")).read()
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties[^\n]*\n\s*(\d+) bytes "
                         r"stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    names = sorted(e[0] for e in entries)
    assert sum("render_kernel" in n for n in names) == 1, names
    assert sorted(int(re.search(r"render_probs_kernelILi(\d+)E", n).group(1)) for n in names
                  if "render_probs_kernel" in n) == [16, 32, 64], names
    for name, stack, st, ld in entries:
        assert (stack, st, ld) == ("0", "0", "0"), name


# ---- refusals --------------------------------------------------------------------------------------------------------
def _probs_args(**k):
    buf = np.zeros(1024, np.uint16)
    p = buf.ctypes.data
    a = dict(probs=p, B=1, C=4, GX=4, GY=4, GZ=2, strides=np.array([8, 2, 1], np.int64), cmap=None, ignore=255,
             empty=0, origin=np.zeros(3), voxel=0.2, V=1, cams=np.r_[np.eye(3).reshape(-1), 0.0, 0.0, -1.0], W=8,
             H=4, near=0.0, far=np.inf, t_min=1e-4, lut=None, cls=p, depth=None, opacity=None, probs_out=None)
    a.update(k)
    keep = [buf] + [v for v in a.values() if isinstance(v, np.ndarray)]
    ptr = lambda v: v.ctypes.data if isinstance(v, np.ndarray) else v      # noqa: E731
    args = (a["probs"], a["B"], a["C"], a["GX"], a["GY"], a["GZ"], ptr(a["strides"]), ptr(a["cmap"]), a["ignore"],
            a["empty"], ptr(a["origin"]), a["voxel"], a["V"], ptr(a["cams"]), a["W"], a["H"], a["near"], a["far"],
            a["t_min"], ptr(a["lut"]), ptr(a["cls"]), ptr(a["depth"]), ptr(a["opacity"]), ptr(a["probs_out"]), None)
    return args, keep


PROBS_BAD = {
    "probs": dict(probs=None), "strides_null": dict(strides=None), "origin_null": dict(origin=None),
    "cams_null": dict(cams=None), "no_output": dict(cls=None), "B0": dict(B=0), "V0": dict(V=0),
    "cameras33": dict(B=3, V=11), "C0": dict(C=0), "C65": dict(C=65), "empty_neg": dict(empty=-1),
    "empty_C": dict(empty=4), "GX": dict(GX=0), "GZ": dict(GZ=-2), "voxels": dict(GX=2048, GY=2048, GZ=512),
    "stride_neg": dict(strides=np.array([8, -2, 1], np.int64)),
    "stride_out": dict(strides=np.array([16, 2, 1], np.int64)), "W0": dict(W=0), "H0": dict(H=0),
    "H_big": dict(H=70000), "voxel0": dict(voxel=0.0), "voxel_nan": dict(voxel=float("nan")),
    "origin_inf": dict(origin=np.array([0.0, np.inf, 0.0])), "cams_nan": dict(cams=np.full(12, np.nan)),
    "ignore": dict(ignore=65536), "near_neg": dict(near=-0.1), "near_inf": dict(near=np.inf),
    "far": dict(near=1.0, far=1.0), "far_nan": dict(far=float("nan")), "t_min_neg": dict(t_min=-0.1),
    "t_min_one": dict(t_min=1.0), "t_min_nan": dict(t_min=float("nan")),
    "align_probs": dict(probs=np.zeros(64, np.uint8).ctypes.data + 1),
    "align_cmap": dict(cmap=np.zeros(64, np.uint8).ctypes.data + 1),
    "align_opacity": dict(opacity=np.zeros(64, np.uint8).ctypes.data + 2),
    "align_probs_out": dict(probs_out=np.zeros(64, np.uint8).ctypes.data + 1),
}


@pytest.mark.parametrize("case", sorted(PROBS_BAD))
def test_render_probs_entry_refusals(case):
    _build.build()
    L = _lib.lib()
    args, keep = _probs_args(**PROBS_BAD[case])
    assert L.occd_render_probs(*args) == _lib.ERR_ARG, case
    assert L.occd_last_error().startswith(b"occd_render_probs: "), L.occd_last_error()


def test_render_probs_refusals(monkeypatch):
    called = []
    monkeypatch.setattr(_lib, "lib", lambda: called.append(1))
    p = torch.zeros(2, 5, 8, 6, 4, dtype=torch.float16)
    m = torch.zeros(2, 8, 6, 4, dtype=torch.uint16)
    E, K = np.eye(4), _K()
    go = lambda **kw: render.render_probs(**dict(dict(probs=p, E=E, K=K, size=(64, 48),   # noqa: E731
                                                      grid_origin=(0, 0, 0), grid_voxel=0.2), **kw))
    with pytest.raises(TypeError, match="float16"):
        go(probs=p.float())
    with pytest.raises(ValueError, match="contiguous"):
        go(probs=p.transpose(2, 3))
    with pytest.raises(ValueError, match="contiguous"):
        go(probs=p[0, 0])
    with pytest.raises(ValueError, match="at most 64"):
        go(probs=torch.zeros(1, 65, 2, 2, 2, dtype=torch.float16))
    with pytest.raises(TypeError, match="class_map must be a uint16"):
        go(class_map=m.int())
    with pytest.raises(ValueError, match="class_map must be contiguous"):
        go(class_map=m[:1])
    with pytest.raises(ValueError, match="class_map must be contiguous"):
        go(class_map=m.transpose(1, 2).contiguous())
    with pytest.raises(ValueError, match="render_probs: empty \\(5\\) must be a channel index below C = 5"):
        go(empty=5)
    with pytest.raises(ValueError, match="empty and ignore"):
        go(ignore=-1)
    with pytest.raises(ValueError, match="axes"):
        go(axes="zyx")
    with pytest.raises(ValueError, match="size"):
        go(size=(0, 48))
    with pytest.raises(ValueError, match="near"):
        go(near=2.0, far=1.0)
    with pytest.raises(ValueError, match="render_probs: E"):
        go(E=np.zeros((4, 4)))
    with pytest.raises(ValueError, match="at most 32 cameras"):
        go(E=np.stack([np.stack([np.eye(4)] * 17)] * 2))
    for t in (-0.1, 1.0, 0.99999999, float("nan")):
        with pytest.raises(ValueError, match="min_transmittance"):
            go(min_transmittance=t)
    with pytest.raises(ValueError, match="inv_map"):
        go(inv_map=np.arange(4))
    shape = (2, 1, 48, 64)
    outs = [torch.empty(shape, dtype=torch.uint16), torch.empty(shape), torch.empty(shape),
            torch.empty((2, 1, 5, 48, 64), dtype=torch.float16)]
    with pytest.raises(ValueError, match="at least one"):
        go(out=render.SoftView(None, None, None, None))
    with pytest.raises(TypeError, match="out.opacity"):
        go(out=render.SoftView(None, None, outs[0], None))
    with pytest.raises(ValueError, match="out.probs"):
        go(out=render.SoftView(None, None, None, torch.empty((2, 1, 4, 48, 64), dtype=torch.float16)))
    # every argument good: the tensors on the CPU are the last refusal before the launch
    with pytest.raises(ValueError, match="CUDA device"):
        go(out=render.SoftView(*outs), class_map=m, inv_map=np.arange(5), min_transmittance=0.0)
    with pytest.raises(ValueError, match="CUDA device"):
        go(empty=4, ignore=7, near=0.5, far=80.0)
    assert not called


def test_scene_map_render_probs_refuses_before_any_launch(monkeypatch):
    called = []
    monkeypatch.setattr(_lib, "lib", lambda: called.append(1))
    from occdepth_b200 import fusion
    monkeypatch.setattr(fusion.SceneMap, "classes", lambda *a, **k: called.append(2))
    m = _cpu_map()
    K = _K()
    with pytest.raises(ValueError, match="SceneMap.render_probs: unknown"):
        m.render_probs(np.eye(4), K, (64, 48), unknown=-1)
    with pytest.raises(ValueError, match="SceneMap.render_probs: min_transmittance"):
        m.render_probs(np.eye(4), K, (64, 48), min_transmittance=1.0)
    with pytest.raises(ValueError, match="SceneMap.render_probs: inv_map"):
        m.render_probs(np.eye(4), K, (64, 48), inv_map=np.arange(3))
    with pytest.raises(ValueError, match="SceneMap.render_probs: E"):
        m.render_probs(np.full((4, 4), np.nan), K, (64, 48))
    with pytest.raises(ValueError, match="SceneMap.render_probs: size"):
        m.render_probs(np.eye(4), K, (0, 48))
    with pytest.raises(ValueError, match="SceneMap.render_probs: near"):
        m.render_probs(np.eye(4), K, (64, 48), near=3.0, far=1.0)
    with pytest.raises(ValueError, match="at most 32"):
        m.render_probs(np.stack([np.eye(4)] * 33)[None], K, (64, 48))
    assert not called


def test_predict_view_soft_refusals(kitti_model, monkeypatch):
    m = kitti_model
    ran = []
    monkeypatch.setattr(m, "_run_frames", lambda *a, **k: ran.append(a))
    monkeypatch.setattr(m, "_run_frame", lambda *a, **k: ran.append(a))
    monkeypatch.setattr(m, "_check_mode", lambda x: None)
    with pytest.raises(ValueError, match="1 to 32 cameras"):
        m.predict_view([_kitti()] * 17, views=(0, 1), soft=True)
    with pytest.raises(ValueError, match="views \\(0, 2\\) of a frame with 2 cameras"):
        m.predict_view(_kitti(), views=(0, 2), soft=True)
    with pytest.raises(ValueError, match="predict_view: near"):
        m.predict_view(_kitti(), near=-1.0, soft=True)
    for t in (-1e-3, 1.0):
        with pytest.raises(ValueError, match="predict_view: min_transmittance"):
            m.predict_view(_kitti(), soft=True, min_transmittance=t)
    with pytest.raises(ValueError, match="inv_map"):
        m.predict_view(_kitti(), soft=True, inv_map=np.arange(3))
    with pytest.raises(ValueError, match="predict_view: E is singular"):
        m.predict_view(_kitti(T=np.stack([np.eye(4), np.zeros((4, 4))])), views=(0, 1), soft=True)
    assert not ran
    assert m.predict_view(_kitti(), soft=True) is None
    assert len(ran) == 1 and ran[0][1:] == (True, None, None, False, True)   # predict_frame's probabilities plan
    from occdepth_b200.parallel import SimSlabGroup
    m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
    try:
        with pytest.raises(NotImplementedError, match="slab"):
            m.predict_view(_kitti(), soft=True)
    finally:
        m.__dict__.pop("slab_ctx", None)
    assert len(ran) == 1
