"""The class-map gather of the slab partition (parallel.GatherRootOp) on 3 CPU ranks with the gloo backend: uneven
slabs of a uint16 map arrive on rank 0 as their concatenation, and the other ranks' buffers are left as they were."""
import os
import socket

import torch.multiprocessing as mp

BOUNDS = [(0, 4), (4, 6), (6, 11)]          # uneven full-resolution X slabs of an 11 x 3 x 5 map
Y, Z = 3, 5


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _slab(rank):
    import torch
    lo, hi = BOUNDS[rank]
    # values above 255 and 32767, so both bytes of every uint16 and its sign bit travel
    v = torch.arange(lo * Y * Z, hi * Y * Z, dtype=torch.int32) * 613 + 40000 * (rank % 2)
    return (v % 65536).to(torch.uint16).view(1, hi - lo, Y, Z)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch
    import torch.distributed as dist
    from occdepth_b200 import parallel
    parallel.init(backend="gloo")
    ctx = parallel.SlabContext(halo=3)
    src = _slab(rank).clone()
    dst = torch.zeros(1, BOUNDS[-1][1], Y, Z, dtype=torch.uint16) if rank == 0 else None
    op = ctx.gather_root_op(src, dst, BOUNDS)
    op.run()
    op.run()                                  # a plan replays the op every frame
    q.put((rank, src.to(torch.int32).tolist(), None if dst is None else dst.to(torch.int32).tolist()))
    dist.destroy_process_group()


def test_gather_root_gloo_uneven_slabs():
    import torch
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    world = len(BOUNDS)
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    whole = torch.cat([_slab(r) for r in range(world)], 1).to(torch.int32).tolist()
    assert res[0][2] == whole
    for r, src, dst in res:
        assert src == _slab(r).to(torch.int32).tolist()
        if r:
            assert dst is None


def test_gather_root_refuses_a_slab_of_the_wrong_size():
    import pytest
    import torch
    from occdepth_b200.parallel import SlabContext
    ctx = SlabContext(rank=1, world=3)
    with pytest.raises(RuntimeError, match="does not hold planes"):
        ctx.gather_root_op(torch.zeros(1, 3, Y, Z, dtype=torch.uint16), None, BOUNDS)
