"""Model files under the X-slab partition: every rank's plan of predict_frame(slab_output="root") exported to its own
file (the rank plans built one after another on one device, parallel.SimSlabGroup contexts), loaded on a local
communicator and run in lock step by occd_model_run_frame_group: rank 0's whole map bit for bit the unpartitioned
predict_frame's, for every case of test_gpu_slab_camera.CASES, with and without the CUDA graph; the label remap and
the confidence; unpartitioned exports unchanged; and, with two GPUs, NCCL between processes and tools/occd_run."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200.parallel import SimSlabGroup

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if d not in sys.path:
        sys.path.insert(0, d)
from camera_frames import kitti_frame, kitti_geometry  # noqa: E402
from test_gpu_slab_camera import CASES, _camera_frames  # noqa: E402


def _sc():
    import shipped_configs
    return shipped_configs


def _same(a, b):
    return a is not None and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def export_ranks(m, world, frame, paths, **kw):
    """every rank's model file of `frame`, the rank plans built one after another on this device"""
    grp = SimSlabGroup(world, halo=3)
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                deploy.export(m, paths[r], frame, slab_output="root", **kw)
    finally:
        m.__dict__.pop("slab_ctx", None)


def load_group(paths):
    comms = deploy.Comm.local(len(paths))
    return [deploy.LoadedModel(p, c) for p, c in zip(paths, comms)]


# the cases that also export the label remap and the confidence: one KITTI, one NYU
REMAP_CONF = {("kitti_b3_f32_flospdepth_2080ti", "tf32", 3), ("nyu_b4_f100_2080ti", "tf32", 2)}


@pytest.mark.parametrize("name,precision,world", CASES)
def test_shipped_config_rank_files_in_lockstep(tmp_path, name, precision, world):
    sc = _sc()
    _free()
    spec = sc.CONFIGS[name]
    m, _, _ = sc.make_case(name)
    m = m.cuda().set_precision(precision)
    frames = _camera_frames(sc, spec)
    with torch.no_grad():
        want = [m.predict_frame(f) for f in frames]
    paths = [tmp_path / ("r%d.occd" % r) for r in range(world)]
    export_ranks(m, world, frames[0], paths)
    models = load_group(paths)
    side = torch.cuda.Stream()
    for graph in (True, False, True):               # the first frame captures, the others replay; one by one; again
        got = [deploy.run_frame_group(models, f, stream=side, graph=graph) for f in frames]
        side.synchronize()
        for i, (g, w) in enumerate(zip(got, want)):
            assert _same(g, w), (graph, i, int((g.int() != w.int()).sum()))
    assert models[0].info().graph == 1
    for x in models:
        x.close()
    if (name, precision, world) in REMAP_CONF:
        inv = np.random.default_rng(5).permutation(256)[:m.n_classes]
        with torch.no_grad():
            want_pairs = [m.predict_frame(f, inv_map=inv, confidence=True) for f in frames]
        export_ranks(m, world, frames[0], paths, inv_map=inv, confidence=True)
        models = load_group(paths)
        for graph in (True, False):
            got = [deploy.run_frame_group(models, f, stream=side, graph=graph, conf=True) for f in frames]
            side.synchronize()
            for i, ((gm, gc_), (wm, wc)) in enumerate(zip(got, want_pairs)):
                assert _same(gm, wm), (graph, i)
                assert _same(gc_, wc), (graph, i)
        for x in models:
            x.close()
    del m
    _free()


def test_unpartitioned_export_is_unchanged(tmp_path):
    """a file exported without the partition has no slab flag and block, loads with occd_model_load and is refused by
    occd_model_load_slab; rank files are refused by occd_model_load, and a local rank does not run alone"""
    sc = _sc()
    hw, full = (96, 320), (64, 64, 16)
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=hw, full=full)
    m = m.cuda()
    f = dict(kitti_frame(2, hw[0], hw[1], 1), **kitti_geometry(hw[0], hw[1], full))
    with torch.no_grad():
        deploy.export(m, tmp_path / "a.occd", f)
        want = m.predict_frame(f)
    a = (tmp_path / "a.occd").read_bytes()
    flags = int(np.frombuffer(a, "<u4", 1, 8 + 4 * 4)[0])
    assert not flags & deploy.FLAG_SLAB
    cm = deploy.LoadedModel(tmp_path / "a.occd")
    assert _same(cm.run_frame(f), want)
    cm.close()
    comm = deploy.Comm.local(1)[0]
    with pytest.raises(RuntimeError, match="holds no X-slab partition"):
        deploy.LoadedModel(tmp_path / "a.occd", comm)
    # a rank file: refused by occd_model_load; a local rank refuses to run alone
    export_ranks(m, 2, f, [tmp_path / "r0.occd", tmp_path / "r1.occd"])
    with pytest.raises(RuntimeError, match="occd_model_load_slab"):
        deploy.LoadedModel(tmp_path / "r0.occd")
    models = load_group([tmp_path / "r0.occd", tmp_path / "r1.occd"])
    with pytest.raises(RuntimeError, match="occd_model_run_frame_group"):
        models[0].run_frame(f)
    with pytest.raises(RuntimeError, match="rank r of one local group"):
        deploy.run_frame_group(models[::-1], f)
    assert _same(deploy.run_frame_group(models, f), want)
    for x in models:
        x.close()
    with pytest.raises(NotImplementedError, match="slab_output='root'"):
        m.__dict__["slab_ctx"] = SimSlabGroup(2, halo=3).ctxs[0]
        try:
            deploy.export(m, tmp_path / "x.occd", f, slab_output="slab")
        finally:
            m.__dict__.pop("slab_ctx", None)
    assert not (tmp_path / "x.occd").exists()


# ---- two GPUs: NCCL between processes ---------------------------------------------------------------------------------
HW, FULL = (96, 320), (128, 128, 16)


def _small_frames():
    geo = kitti_geometry(HW[0], HW[1], FULL)
    return [dict(kitti_frame(2, HW[0], HW[1], s), **geo) for s in (1, 2)] + \
        [dict(kitti_frame(2, HW[0], HW[1], 3, shift=0.3), **geo)]


def _nccl_lib():
    """the libnccl.so.2 this process has loaded (torch's)"""
    torch.cuda.init()
    with open("/proc/self/maps") as fh:
        for line in fh:
            if "libnccl.so" in line:
                return line.split()[-1]
    return None


def _nccl_worker(rank, world, tmp, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from occdepth_b200 import parallel
    try:
        torch.cuda.set_device(rank)
        sc = _sc()
        m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=HW, full=FULL)   # seeded: equal on every rank
        m = m.cuda()
        frames = _small_frames()
        with torch.no_grad():
            want = [m.predict_frame(f).cpu() for f in frames] if rank == 0 else None
            m.enable_slab_parallel(parallel.SlabContext(halo=3))
            path = os.path.join(tmp, "r%d.occd" % rank)
            deploy.export(m, path, frames[0], slab_output="root")
        id_path = os.path.join(tmp, "nccl.id")
        if rank == 0:
            with open(id_path + ".tmp", "wb") as fh:
                fh.write(deploy.Comm.unique_id())
            os.rename(id_path + ".tmp", id_path)
        else:
            import time
            for _ in range(3000):
                if os.path.exists(id_path):
                    break
                time.sleep(0.1)
        with open(id_path, "rb") as fh:
            comm = deploy.Comm(fh.read(), rank, world)
        cm = deploy.LoadedModel(path, comm)
        ok = True
        for graph in (True, False):
            got = [cm.run_frame(f, graph=graph) for f in frames]
            torch.cuda.synchronize()
            if rank == 0:
                ok = ok and all(_same(g.cpu(), w) for g, w in zip(got, want))
            else:
                ok = ok and all(g is None for g in got)
        cm.close()
        comm.close()
        q.put((rank, ok, None))
    except Exception as e:  # noqa: BLE001 -- reported to the parent
        q.put((rank, False, repr(e)))


def _join(procs, timeout):
    """wait for the workers; any still alive after `timeout` seconds is terminated"""
    for p in procs:
        p.join(timeout)
    for p in procs:
        if p.is_alive():
            p.terminate()
            p.join(30)


def test_rank_files_over_nccl(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("two GPUs are needed for the NCCL run (%d visible)" % torch.cuda.device_count())
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = sorted(q.get(timeout=900) for _ in range(2))
    finally:
        _join(procs, 120)
    assert all(r[2] is None for r in res), res
    assert all(r[1] for r in res), res
    assert all(p.exitcode == 0 for p in procs)
    # tools/occd_run on both ranks: rank 0 writes the same .label bytes as predict_frame's maps
    frames = _small_frames()
    with open(tmp_path / "imgs.u8", "wb") as fi, open(tmp_path / "calib.f64", "wb") as fc:
        for f in frames:
            fi.write(np.ascontiguousarray(f["img"], np.uint8).tobytes())
            fc.write(np.ascontiguousarray(f["cam_k"], np.float64).tobytes())
            fc.write(np.ascontiguousarray(f["T_velo_2_cam"], np.float64).tobytes())
    sc = _sc()
    m, _, _ = sc.make_case("kitti_b3_f32_flospdepth_2080ti", img_hw=HW, full=FULL)
    m = m.cuda()
    with torch.no_grad():
        want = [m.predict_frame(f) for f in frames]
    lib = _nccl_lib()
    out = tmp_path / "labels"
    out.mkdir()
    H0, W0 = frames[0]["img"].shape[1:3]
    cmds = []
    for r in range(2):
        cmd = [_build.occd_run_path(), str(tmp_path / ("r%d.occd" % r)), str(tmp_path / "imgs.u8"),
               str(tmp_path / "calib.f64"), str(len(frames)), str(out), "--raw", str(H0), str(W0), "--world", "2",
               "--rank", str(r), "--nccl-id", str(tmp_path / "run.id")] + (["--nccl-lib", lib] if lib else [])
        cmds.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                                     env=dict(os.environ, CUDA_VISIBLE_DEVICES=str(r))))
    outs = []
    try:
        for p in cmds:
            outs.append(p.communicate(timeout=600)[0])
    finally:
        for p in cmds:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert all(p.returncode == 0 for p in cmds), outs
    for i, w in enumerate(want):
        assert (out / ("%06d.label" % i)).read_bytes() == w.cpu().numpy().tobytes(), i
