"""Camera frames under the X-slab partition: `occd_vox2pix_range_fwd` against the slice of the whole-grid indices; every
shipped configuration's rank plans (parallel.SimSlabGroup, lock-step on one GPU) staged from camera frames, against
the unpartitioned `predict_frame` bit for bit; the public entry points (`predict_frame`, `predict_voxels`,
`CameraPipeline` with `slab_output`) driven from one thread per rank; a two-process NCCL run of the pipeline; and the
refusals."""
import copy
import gc
import os
import sys
import threading

import numpy as np
import pytest
import torch

from occdepth_b200 import _lib
from occdepth_b200 import data as D
from occdepth_b200.parallel import SimSlabContext, SimSlabGroup

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
from camera_frames import kitti_frame, kitti_geometry, nyu_frame  # noqa: E402

GOLD = torch.load(os.path.join(ROOT, "tests", "golden", "vox2pix.pt"))


def _sc():
    import shipped_configs
    return shipped_configs


def _u16_equal(a, b):
    return a is not None and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _free():
    gc.collect()
    torch.cuda.empty_cache()


# ---- 1. the windowed index kernel -----------------------------------------------------------------------------------
@pytest.mark.parametrize("f32", [False, True], ids=["f64_pose", "f32_pose"])
@pytest.mark.parametrize("name,pattern_id", [("kitti_p0", 0), ("kitti_p3", 3), ("nyu_p8", 0), ("nyu_p8", 8)])
def test_vox2pix_range_is_the_slice_of_the_whole_grid(name, pattern_id, f32):
    c = GOLD[name]
    E = c["cam_E"].numpy().astype(np.float32 if f32 else np.float64)
    args = (E, c["cam_k"].numpy(), c["vox_origin"].numpy(), c["voxel_size"], c["img_W"], c["img_H"], c["scene_size"],
            pattern_id)
    X, Y, Z = (int(v) for v in D.volume_dims(c["vox_origin"].numpy(), c["voxel_size"], c["scene_size"]))
    plane, N = Y * Z, X * Y * Z
    pix, fov, z = D.vox2pix(*args)
    P = pix.shape[1]
    for v0, n in ((0, N), (0, 2 * plane), (N // 3, N // 3 + 7), ((X // 2) * plane, plane), (N - plane, plane),
                  (N - N // 4, N // 4), (N - 1, 1)):
        wp = torch.full((n, P, 2), -7, dtype=torch.int64, device="cuda")
        wf = torch.ones(n, P, dtype=torch.bool, device="cuda")
        wz = torch.full((n,), float("nan"), dtype=z.dtype, device="cuda")
        D.vox2pix_into(wp, wf, wz, *args, voxel_range=(v0, n))
        assert torch.equal(wp, pix[v0:v0 + n]) and torch.equal(wf, fov[v0:v0 + n]), (v0, n)
        assert torch.equal(wz.view(torch.int32 if f32 else torch.int64),
                           z[v0:v0 + n].view(torch.int32 if f32 else torch.int64)), (v0, n)


def test_vox2pix_range_refuses_windows_outside_the_grid():
    c = GOLD["kitti_p0"]
    args = (c["cam_E"].numpy(), c["cam_k"].numpy(), c["vox_origin"].numpy(), c["voxel_size"], c["img_W"], c["img_H"],
            c["scene_size"], 0)
    N = c["pix"].shape[0]
    pix = torch.zeros(8, 1, 2, dtype=torch.int64, device="cuda")
    fov = torch.zeros(8, 1, dtype=torch.bool, device="cuda")
    z = torch.zeros(8, dtype=torch.float64, device="cuda")
    for window in ((N - 4, 8), (-1, 8), (0, 0)):
        with pytest.raises(ValueError, match="voxel_range"):
            D.vox2pix_into(pix, fov, z, *args, voxel_range=window)
    E = np.ascontiguousarray(c["cam_E"].numpy())
    k = np.ascontiguousarray(c["cam_k"].numpy().astype(np.float32))
    o = np.ascontiguousarray(c["vox_origin"].numpy().astype(np.float32))
    pat = np.zeros(2, np.int32)
    X, Y, Z = (int(v) for v in D.volume_dims(c["vox_origin"].numpy(), c["voxel_size"], c["scene_size"]))
    for v0, n in ((N - 4, 8), (-1, 8), (0, 0), (N, 1)):
        rc = _lib.lib().occd_vox2pix_range_fwd(E.ctypes.data, 0, k.ctypes.data, o.ctypes.data, c["voxel_size"], X, Y, Z,
                                               c["img_W"], c["img_H"], pat.ctypes.data, 1, pix.data_ptr(),
                                               fov.data_ptr(), z.data_ptr(), v0, n, _lib.stream_ptr())
        assert rc == _lib.ERR_ARG and b"window" in _lib.lib().occd_last_error(), (v0, n)
    torch.cuda.synchronize()


# ---- 2. every shipped configuration, rank plans in lock-step ---------------------------------------------------------
CASES = [("kitti_b3_f32_flospdepth_2080ti", "tf32", 2), ("kitti_b3_f32_flospdepth_2080ti", "tf32", 3),
         ("kitti_b3_f32_flospdepth_2080ti", "tf32", 8), ("kitti_b3_f32_flospdepth_2080ti", "bf16", 2),
         ("kitti_b3_f24_flospdepth_mono_2080ti", "tf32", 2), ("kitti_b3_f24_flospdepth_mono_2080ti", "tf32", 10),
         ("kitti_b7_f64_flosp_a100", "tf32", 2), ("kitti_b7_f64_flospdepth_a100", "tf32", 3),
         ("nyu_b4_f100_2080ti", "tf32", 2), ("nyu_b4_f100_2080ti", "tf32", 3), ("nyu_b4_f100_2080ti", "tf32", 5),
         ("nyu_b4_f100_2080ti", "bf16", 3), ("nyu_b7_f200_v100", "tf32", 2)]


def _camera_frames(sc, spec):
    """three frames: KITTI repeats the first calibration in the second and changes it in the third; every NYU frame
    has its own pose"""
    if spec["dataset"] == "NYU":
        frames = [nyu_frame(1), nyu_frame(2), nyu_frame(3)]
        frames[1]["cam_pose"][0, 3] += 0.2
        return [dict(f, img_hw=sc.NYU_IMG) for f in frames]
    H, W = sc.KITTI_IMG
    geo = kitti_geometry(H, W, sc.KITTI_FULL)
    frames = [kitti_frame(spec["views"], H, W, 1), kitti_frame(spec["views"], H, W, 2),
              kitti_frame(spec["views"], H, W, 3, shift=0.3)]
    return [dict(f, **geo) for f in frames]


def _rank_entries(m, world, f, classes):
    """the rank plans of camera frame `f` (m._frame_inputs) built as the partitioned predict_frame builds them"""
    grp = SimSlabGroup(world, halo=3)
    dev = f["imgs"].device
    ents = []
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad(), torch.cuda.device(dev):
                ents.append(m._build(1, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["batch"], classes=classes))
    finally:
        m.__dict__.pop("slab_ctx", None)
    return ents


def _run_ranks(m, ents, f):
    for e in ents:
        m._stage_frame(e, f)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    torch.cuda.synchronize()


@pytest.mark.parametrize("name,precision,world", CASES)
def test_shipped_config_frames_partitioned(monkeypatch, name, precision, world):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    _free()
    spec = sc.CONFIGS[name]
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    frames = _camera_frames(sc, spec)
    inv = np.random.default_rng(5).permutation(256)[:m.n_classes]
    with torch.no_grad():
        want = [m.predict_frame(f) for f in frames]
        want_inv = m.predict_frame(frames[2], inv_map=inv)
        want_logits = m.predict_frame(frames[0], classes=False)["ssc_logit"]
    m.invalidate_plans()
    dev = next(m.parameters()).device
    fs = [m._frame_inputs(f, dev) for f in frames]
    # "slab": the ranks' maps concatenate to the whole; vox2pix runs on every rank for a new calibration only
    calls = []
    orig = D.vox2pix_into
    monkeypatch.setattr(D, "vox2pix_into", lambda *a, **k: (calls.append(k.get("voxel_range")), orig(*a, **k))[1])
    ents = _rank_entries(m, world, fs[0], ("classes", None))
    per_frame = []
    for i, f in enumerate(fs):
        n0 = len(calls)
        _run_ranks(m, ents, f)
        per_frame.append(len(calls) - n0)
        got = torch.cat([e[4] for e in ents], 1)
        assert _u16_equal(got, want[i]), (i, int((got.int() != want[i].int()).sum()))
    VL = 2 if (spec["views"] == 2 or spec["dataset"] == "NYU") else 1
    if spec["dataset"] == "NYU":
        assert per_frame == [world * VL] * 3
    else:
        assert per_frame == [world * VL, 0, world * VL]
    windows = sorted(set(calls))
    assert len(windows) == world and windows[0][0] == 0 and all(n > 0 for _, n in windows)
    assert sum(n for _, n in windows) == fs[0]["N"]               # the windows tile the grid
    del ents
    _free()
    # "root", with an inv_map: rank 0 holds the whole map, the other ranks nothing
    ents = _rank_entries(m, world, fs[2], ("classes", m._class_lut(inv), "root"))
    _run_ranks(m, ents, fs[2])
    assert _u16_equal(ents[0][4], want_inv)
    assert all(e[4] is None for e in ents[1:])
    assert [op.name for op in ents[0][0].ops].count("gather_root") == 1
    del ents
    _free()
    # classes=False, "slab": the logits
    ents = _rank_entries(m, world, fs[0], None)
    _run_ranks(m, ents, fs[0])
    got = torch.cat([m._outputs(e)["ssc_logit"] for e in ents], 2)
    assert _bits_equal(got, want_logits)
    del ents, m
    _free()


# ---- 3. the public entry points, one model replica per rank, driven from threads -----------------------------------
class _Waiting:
    """a simulated communication op that first waits for every rank to reach it (the ranks share one stream, so the
    peers' earlier launches are enqueued before its copies), and keeps the peers from running ahead until it is done"""

    def __init__(self, op, barrier):
        self.op, self.barrier, self.name, self.flops = op, barrier, op.name, 0

    def run(self, stream=None):
        self.barrier.wait()
        self.op.run(stream)
        self.barrier.wait()


class _ThreadSlabContext(SimSlabContext):
    def exchange_op(self, cl):
        return _Waiting(super().exchange_op(cl), self.group.barrier)

    def all_gather_op(self, src, dst):
        return _Waiting(super().all_gather_op(src, dst), self.group.barrier)

    def gather_root_op(self, src, dst, bounds):
        return _Waiting(super().gather_root_op(src, dst, bounds), self.group.barrier)


class _ThreadSlabGroup(SimSlabGroup):
    def __init__(self, world):
        super().__init__(world, halo=3)
        self.barrier = threading.Barrier(world, timeout=600)
        self.ctxs = [_ThreadSlabContext(self, r, world, 3) for r in range(world)]


def _vox(vl):
    """numpy copy of frame 0 of a VoxelList: counts, histogram and the written rows"""
    count = vl.counts()[0]
    t = int(count.sum())
    return dict(count=count, hist=vl.hist[0].cpu().numpy(), index=vl.index[0, :t].cpu().numpy(),
                cls=vl.cls[0, :t].cpu().numpy(), xyz=vl.xyz[0, :t].cpu().numpy())


def _run_threads(world, fn, barrier):
    errors = []

    def body(r):
        try:
            fn(r)
        except BaseException as e:  # noqa: BLE001 -- re-raised below; free the peers waiting on the barrier
            errors.append(e)
            barrier.abort()
    threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]


@pytest.mark.parametrize("world", [2, 3])        # 2: the views sharded; 3: both views on every rank, uneven slabs
def test_public_entry_points_from_rank_threads(monkeypatch, world):
    from occdepth_b200.serving import CameraPipeline
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    sc = _sc()
    _free()
    hw, full = (96, 320), (128, 128, 16)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    replicas = [copy.deepcopy(m).cuda() for _ in range(world)]
    m = m.cuda()
    geo = kitti_geometry(hw[0], hw[1], full)
    frames = [kitti_frame(2, hw[0], hw[1], 1), kitti_frame(2, hw[0], hw[1], 2),
              kitti_frame(2, hw[0], hw[1], 3, shift=0.3)]
    f0 = dict(frames[0], **geo)
    inv = np.arange(20)[::-1].copy()
    with torch.no_grad():
        want = [m.predict_frame(dict(f, **geo)).cpu() for f in frames]
        want_inv = m.predict_frame(f0, inv_map=inv).cpu()
        want_logits = m.predict_frame(f0, classes=False)["ssc_logit"].cpu()
        want_vox = _vox(m.predict_voxels(f0))
    grp = _ThreadSlabGroup(world)
    res = [dict() for _ in range(world)]

    def rank(r):
        mr = replicas[r].enable_slab_parallel(grp.ctxs[r])
        out = res[r]
        with torch.no_grad():
            out["slab"] = [mr.predict_frame(dict(f, **geo), slab_output="slab").cpu() for f in frames]
            y = mr.predict_frame(f0, inv_map=inv, slab_output="root")
            out["root"] = None if y is None else y.cpu()
            out["logits"] = mr.predict_frame(f0, classes=False, slab_output="slab")["ssc_logit"].cpu()
            vl = mr.predict_voxels(f0, slab_output="root")
            out["vox_root"] = None if vl is None else _vox(vl)
            out["vox_slab"] = _vox(mr.predict_voxels(f0, slab_output="slab"))
            pipe = CameraPipeline(mr, slab_output="root", **geo)
            got = {}
            for f in frames:
                t = pipe.submit(f)
                if t is not None:
                    got[t] = pipe.result(t)
                    got[t] = None if got[t] is None else got[t].clone()
                out["h2d"] = pipe.h2d_bytes
            t = pipe.flush()
            r_last = pipe.result(t)
            got[t] = None if r_last is None else r_last.clone()
            out["pipe"] = got
    _run_threads(world, rank, grp.barrier)
    for i, w in enumerate(want):
        assert _u16_equal(torch.cat([res[r]["slab"][i] for r in range(world)], 1), w), i
    assert _u16_equal(res[0]["root"], want_inv) and all(res[r]["root"] is None for r in range(1, world))
    assert _bits_equal(torch.cat([res[r]["logits"] for r in range(world)], 2), want_logits)
    # predict_voxels: "root" is the unpartitioned list; "slab" lists concatenate, in-FOV rows first, in rank order
    vr = res[0]["vox_root"]
    for k in want_vox:
        assert np.array_equal(vr[k], want_vox[k]), k
    assert all(res[r]["vox_root"] is None for r in range(1, world))
    parts = [res[r]["vox_slab"] for r in range(world)]
    n_in = [int(p["count"][0]) for p in parts]
    assert np.array_equal(sum(p["count"] for p in parts), want_vox["count"])
    assert np.array_equal(sum(p["hist"] for p in parts), want_vox["hist"])
    for k in ("index", "cls", "xyz"):
        cat = np.concatenate([p[k][:n] for p, n in zip(parts, n_in)] + [p[k][n:] for p, n in zip(parts, n_in)])
        assert np.array_equal(cat, want_vox[k]), k
    # the pipeline: rank 0 reads back the whole maps, the other ranks nothing; a view-sharded rank copies one view
    assert sorted(res[0]["pipe"]) == [0, 1, 2]
    for i, w in enumerate(want):
        assert _u16_equal(res[0]["pipe"][i], w), i
    assert all(v is None for r in range(1, world) for v in res[r]["pipe"].values())
    img_bytes = frames[0]["img"].nbytes
    for r in range(world):
        assert res[r]["h2d"] == (img_bytes // 2 if world % 2 == 0 else img_bytes), r
        assert replicas[r].slab_view(2) == (r // (world // 2) if world % 2 == 0 else None)
    del replicas, m
    _free()


# ---- 4. two processes over NCCL ---------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from occdepth_b200 import parallel
    from occdepth_b200.serving import CameraPipeline
    try:
        torch.cuda.set_device(rank)
        parallel.init(backend="nccl", device=torch.device("cuda", rank))
        sc = _sc()
        hw, full = (96, 320), (128, 128, 16)
        m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)   # seeded: equal on every rank
        m = m.cuda()
        geo = kitti_geometry(hw[0], hw[1], full)
        frames = [kitti_frame(2, hw[0], hw[1], s) for s in (1, 2)] + [kitti_frame(2, hw[0], hw[1], 3, shift=0.3)]
        with torch.no_grad():
            want = [m.predict_frame(dict(f, **geo)).cpu() for f in frames] if rank == 0 else None
            m.enable_slab_parallel(parallel.SlabContext(halo=3))
            pipe = CameraPipeline(m, slab_output="root", **geo)
            got = {}
            for f in frames:
                t = pipe.submit(f)
                if t is not None:
                    r = pipe.result(t)
                    got[t] = None if r is None else r.clone()
            t = pipe.flush()
            r = pipe.result(t)
            got[t] = None if r is None else r.clone()
        ok = all(_u16_equal(got[i], want[i]) for i in range(3)) if rank == 0 else all(v is None for v in got.values())
        q.put((rank, ok, sorted(got), pipe.h2d_bytes, None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001 -- reported to the parent
        q.put((rank, False, [], 0, repr(e)))


def test_camera_pipeline_root_over_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("two GPUs are needed for the NCCL run (%d visible)" % torch.cuda.device_count())
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=900) for _ in range(2))
    for p in procs:
        p.join(120)
    assert all(r[4] is None for r in res), res
    assert all(r[1] and r[2] == [0, 1, 2] for r in res), res
    assert all(p.exitcode == 0 for p in procs)


# ---- 5. refusals --------------------------------------------------------------------------------------------------------
def test_refusals(tmp_path):
    from occdepth_b200 import deploy
    from occdepth_b200.serving import CameraPipeline
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    geo = kitti_geometry(hw[0], hw[1], full)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    m = m.cuda()
    f = dict(kitti_frame(2, hw[0], hw[1], 0), **geo)
    with torch.no_grad():
        for bad in ("slab", "root"):                 # no partition: slab_output must stay None
            with pytest.raises(ValueError, match="enable_slab_parallel"):
                m.predict_frame(f, slab_output=bad)
            with pytest.raises(ValueError, match="enable_slab_parallel"):
                m.predict_voxels(f, slab_output=bad)
            with pytest.raises(ValueError, match="enable_slab_parallel"):
                CameraPipeline(m, slab_output=bad, **geo)
        m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        try:
            with pytest.raises(NotImplementedError, match="slab_output"):
                m.predict_frame(f)
            with pytest.raises(NotImplementedError, match="slab_output"):
                CameraPipeline(m, **geo)
            with pytest.raises(ValueError, match="slab_output must be"):
                m.predict_frame(f, slab_output="whole")
            with pytest.raises(ValueError, match="slab_output must be"):
                CameraPipeline(m, slab_output="whole", **geo)
            with pytest.raises(ValueError, match="classes=True"):
                m.predict_frame(f, classes=False, slab_output="root")
            with pytest.raises(ValueError, match="classes=True"):
                CameraPipeline(m, classes=False, slab_output="root", **geo)
            with pytest.raises(NotImplementedError, match="one frame"):
                m.predict_frame(dict(f, img=np.stack([f["img"]] * 2)), slab_output="slab")
            with pytest.raises(NotImplementedError, match="enable_slab_parallel"):
                deploy.export(m, tmp_path / "x.occd", f)
        finally:
            m.__dict__.pop("slab_ctx", None)
        mi, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full, infer_mode=True)
        mi = mi.cuda()
        mi.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        with pytest.raises(NotImplementedError, match="infer_mode"):
            mi.predict_frame(f, slab_output="slab")
        spec = dict(dataset="NYU", backbone_2d_name="tf_efficientnet_b3_ns", feature=16, trans_2d_to_3d="flosp_depth",
                    views=1, context_prior=False, cascade_cls=False, use_depth_gt=True)
        mn, _, _ = sc.make_case(spec=spec)
        mn = mn.cuda()
        mn.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        with pytest.raises(NotImplementedError, match="FlospDepth"):
            mn.predict_frame(dict(nyu_frame(1), img_hw=sc.NYU_IMG), slab_output="root")
    assert not (tmp_path / "x.occd").exists()
    del m, mi, mn
    _free()
