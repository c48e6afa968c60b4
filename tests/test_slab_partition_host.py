"""The X-slab partition rule (parallel.slab_bounds) and the slab plans of the shipped configurations, on the host:
boundaries on multiples of 2^stages, at least `halo` planes per rank at every exchanging level, the even split
wherever it already worked, the padded CRP all-gather of uneven shards, the refusal that names the largest usable
world size, the argument checks of the windowed frustum entry points, and the halo exchange between slabs of
different depth on gloo ranks."""
import contextlib
import io
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture()
def simt(monkeypatch):
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")


def test_partition_equals_the_even_split_where_that_works():
    from occdepth_b200.parallel import SlabContext, slab_bounds
    for n in range(1, 130):
        for world in range(1, 9):
            if n % world:
                continue
            even = [SlabContext(rank=r, world=world).slab(n) for r in range(world)]
            assert slab_bounds(n, world) == even, (n, world)                 # unit 1, no halo rule
            for stages in (1, 2, 3):
                if n % (world << stages) == 0 and (n // world) >> 2 >= 3:
                    assert slab_bounds(n, world, stages, 3, 3) == even, (n, world, stages)


def test_partition_rules_hold_wherever_a_partition_is_returned():
    from occdepth_b200.parallel import level_planes, slab_bounds
    for n in (12, 24, 36, 60, 64, 100, 128, 256):
        for stages in (2, 3):
            A = 1 << stages
            for world in range(1, 13):
                try:
                    b = slab_bounds(n, world, stages, 3, 3)
                except NotImplementedError as e:
                    assert "largest world size that works for this grid is" in str(e)
                    continue
                assert b[0][0] == 0 and b[-1][1] == n and len(b) == world
                assert all(b[i][1] == b[i + 1][0] for i in range(world - 1))
                assert all(lo % A == 0 for lo, _ in b)                       # boundaries on multiples of A
                units = [(hi - lo) // A for lo, hi in b[:-1]] + [(b[-1][1] - b[-1][0]) // A]
                assert max(units) - min(units) <= 1                          # dealt out as evenly as possible
                assert units == sorted(units, reverse=True)                  # the first ranks take the extra unit
                if world > 1:
                    for k in range(3):
                        assert min(level_planes(lo, hi, k) for lo, hi in b) >= 3, (n, world, stages, k)


def test_nyu_bounds_and_the_refusal_at_eight_ranks():
    from occdepth_b200.parallel import SlabContext, slab_bounds
    for stages in (2, 3):                  # without / with the CRP mega-context conv
        assert slab_bounds(60, 2, stages, 3, 3) == [(0, 32), (32, 60)]
        assert slab_bounds(60, 4, stages, 3, 3) == [(0, 16), (16, 32), (32, 48), (48, 60)]
    with pytest.raises(NotImplementedError, match="largest world size that works for this grid is 4"):
        slab_bounds(60, 8, 3, 3, 3)
    with pytest.raises(NotImplementedError, match="largest world size that works for this grid is 5"):
        slab_bounds(60, 8, 2, 3, 3)
    ctx = SlabContext(rank=3, world=4, halo=3)
    assert ctx.partition(60, 3) == (48, 60)
    assert ctx.level_bounds(15) == [(0, 4), (4, 8), (8, 12), (12, 15)]     # the 1/16 level of the NYU UNet
    assert ctx.level_bounds(30) == [(0, 8), (8, 16), (16, 24), (24, 30)]


def _make(name):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from shipped_configs import make_case
    finally:
        sys.path.pop(0)
    return make_case(name)


def _rank_plans(m, batch, world):
    from occdepth_b200.parallel import SimSlabGroup
    img = batch["img"]
    B, V, _, H, W = img.shape
    pp = batch["projected_pix_%d" % m.project_scale]
    grp = SimSlabGroup(world, halo=3)
    ents = []
    try:
        for ctx in grp.ctxs:
            m.__dict__["slab_ctx"] = ctx
            with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
                ents.append(m._build(B, V, H, W, pp[0].shape[1], pp[0].shape[2], torch.device("cpu"), batch))
    finally:
        m.__dict__.pop("slab_ctx", None)
    return grp, ents


@pytest.mark.parametrize("world,shards", [(2, (4, 3)), (4, (2, 2, 2, 1))])
def test_nyu_crp_plans_pad_the_mega_context_gather(simt, world, shards):
    """NYU with the CRP (60 X planes, 1/16 level 15, mega-context 7 planes): uneven mega-context shards are gathered
    padded to the largest one and transposed into the bmm operand shard by shard"""
    m, batch, _ = _make("nyu_b7_f200_v100")
    grp, ents = _rank_plans(m, batch, world)
    ops = [[getattr(op, "name", "") for op in e[0].ops] for e in ents]
    assert all(o == ops[0] for o in ops)                                     # identical op sequences
    assert ops[0].count("all_gather") == 1 and ops[0].count("occd_cl_transpose") == world
    cd = max(shards)
    for r, (e, ctx) in enumerate(zip(ents, grp.ctxs)):
        gather = next(op for op in e[0].ops if getattr(op, "name", "") == "all_gather")
        assert tuple(gather.src.shape[:2]) == (1, cd) and tuple(gather.dst.shape[:2]) == (1, cd * world)
        assert ctx.n_exchanges == grp.ctxs[0].n_exchanges > 0
        lo, hi = ctx.bounds[r]
        assert tuple(e[4]["ssc_logit"].shape) == (1, 12, hi - lo, 36, 60) and e[6] == lo * 36 * 60
        l16 = ctx.level_bounds(15)[r]
        assert tuple(e[4]["P_logits"].shape) == (1, 4, 7 * 4 * 7, (l16[1] - l16[0]) * 9 * 15)
    mega = [e[4]["P_logits"].shape[3] for e in ents]
    assert sum(mega) == 15 * 9 * 15


@pytest.mark.parametrize("name,world,bounds,shards", [
    ("kitti_b7_f64_flosp_a100", 3, [(0, 48), (48, 88), (88, 128)], (6, 5, 5)),
    ("kitti_b3_f32_flospdepth_2080ti", 6, [(0, 24), (24, 48), (48, 72), (72, 96), (96, 112), (112, 128)],
     (3, 3, 3, 3, 2, 2))])
def test_kitti_crp_plans_on_uneven_slabs(simt, name, world, bounds, shards):
    """KITTI with the CRP (128 X planes in 16 units of 8) over a world size that does not divide them: the ranks
    build identical op sequences, and the mega-context conv (padding 1) gives shards of 2 planes per unit, gathered
    padded to the largest"""
    m, batch, _ = _make(name)
    grp, ents = _rank_plans(m, batch, world)
    assert grp.ctxs[0].bounds == bounds
    ops = [[getattr(op, "name", "") for op in e[0].ops] for e in ents]
    assert all(o == ops[0] for o in ops)
    assert ops[0].count("occd_cl_transpose") == world
    assert len({ctx.n_exchanges for ctx in grp.ctxs}) == 1
    for r, e in enumerate(ents):
        gather = [op for op in e[0].ops if getattr(op, "name", "") == "all_gather"][-1]
        assert tuple(gather.src.shape[:2]) == (1, max(shards))
        mega = [op for op in e[0].ops if getattr(op, "name", "") == "crp.mega_context"][0]
        assert mega._keep[1].dims[1] == shards[r]                           # its output CL: this rank's shard
        lo, hi = bounds[r]
        assert tuple(e[4]["ssc_logit"].shape) == (1, 20, 2 * (hi - lo), 256, 32)
        assert tuple(e[4]["P_logits"].shape) == (1, 4, 16 * 16 * 2, (hi - lo) // 4 * 32 * 4)


def test_occdepth_refusals(simt):
    m, batch, _ = _make("nyu_b7_f200_v100")
    with pytest.raises(NotImplementedError, match="largest world size that works for this grid is 4"):
        _rank_plans(m, batch, 8)
    m, batch, _ = _make("kitti_b3_f24_flospdepth_mono_2080ti")
    batch = dict(batch, img=batch["img"].repeat(2, 1, 1, 1, 1))
    with pytest.raises(NotImplementedError, match="batch size 1"):
        _rank_plans(m, batch, 2)


def test_flospdepth_plan_runs_depthnet_whole_and_samples_the_window(simt):
    """released KITTI model at 2 ranks (view sharding): both views' 1_8 maps are copied out of the all-gather for
    DepthNet, and the frustum sampling covers this rank's 64 of 128 X planes"""
    m, batch, _ = _make("kitti_b3_f32_flospdepth_2080ti")
    grp, ents = _rank_plans(m, batch, 2)
    for r, e in enumerate(ents):
        names = [getattr(op, "name", "") for op in e[0].ops]
        assert names.count("depthnet.gather_views") == 2
        assert names.index("all_gather") < names.index("depthnet.gather_views") < names.index("depthnet.reduce")
        st = e[0].flosp_state
        assert st["window"] == (64 * r, 64) and tuple(st["prob"].shape[:2]) == (1, 2)
        assert grp.ctxs[r].n_exchanges == 24


def test_window_entry_points_refuse_bad_windows_without_a_device():
    from occdepth_b200 import _build, _lib
    _build.build()
    L = _lib.lib()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    X, Y, Z = 8, 4, 2
    for x0, xl in ((0, 0), (-1, 2), (7, 2), (8, 1), (0, 9)):
        rc = L.occd_frustum_sample_window_fwd(p, p, 1, 4, 2, 2, X, Y, Z, x0, xl, 8.0, 8.0, 1.0, 10.0, 1, p, 0, None)
        assert rc != 0 and b"window" in L.occd_last_error(), (x0, xl)
        rc = L.occd_grid_sample_prior_window_fwd(p, p, 1, 4, 2, 2, X, Y, Z, x0, xl, 1, p, 1, None)
        assert rc != 0 and b"window" in L.occd_last_error(), (x0, xl)
    assert L.occd_frustum_sample_window_fwd(None, p, 1, 4, 2, 2, X, Y, Z, 0, 1, 8.0, 8.0, 1.0, 10.0, 1, p, 0,
                                            None) != 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


DEPTHS = (4, 6, 3)


def _uneven_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from occdepth_b200 import parallel
    from occdepth_b200.engine import CL
    parallel.init(backend="gloo")
    ctx = parallel.SlabContext(halo=3)
    n = DEPTHS[rank]
    cl = CL(torch.zeros(1, n + 6, 2, 3, 8, dtype=torch.bfloat16), 8, 0, 3, n)
    lo = sum(DEPTHS[:rank])
    for p in range(n):      # global plane g holds the value g + 1
        cl.buf[0, 3 + p] = lo + p + 1
    ctx.exchange_op(cl).run()
    q.put((rank, cl.buf[0, :, 0, 0, 0].float().tolist()))
    dist.destroy_process_group()


def test_halo_exchange_between_slabs_of_different_depth_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    world = len(DEPTHS)
    procs = [ctx.Process(target=_uneven_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    # global planes 1..13 over slabs of 4, 6 and 3 planes: every margin holds its neighbour's 3 nearest planes
    assert res[0][1] == [0, 0, 0, 1, 2, 3, 4, 5, 6, 7]
    assert res[1][1] == [2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13]
    assert res[2][1] == [8, 9, 10, 11, 12, 13, 0, 0, 0]
