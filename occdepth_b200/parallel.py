"""Multi-GPU plumbing for the forward path: one process per GPU, frames sharded across ranks.

Frames are independent (SURVEY.md section 8e): the data path needs NO collective -- every rank runs the whole
forward on its own frames.  torch.distributed (NCCL on GPUs, gloo in the CPU tests) is used only for the
barrier around a timed region, the max-over-ranks reduction of device times and for gathering predictions.
"""
import ctypes as C
import os

import torch
import torch.distributed as dist

from . import _lib


def env_world():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def init(backend=None, device=None):
    """Initialise the default process group from the torchrun environment (no-op for world size 1)."""
    world, rank, local = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl" and device is not None:
            kw["device_id"] = device
        dist.init_process_group(backend, **kw)
    return world, rank, local


def frame_shard(n_frames, rank, world):
    """Contiguous, balanced shard [lo, hi) of n_frames for `rank` (first n_frames % world ranks get one extra)."""
    base, extra = divmod(n_frames, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def barrier():
    if dist.is_initialized():
        dist.barrier()


def max_over_ranks(value, device=None):
    """max of a python float over all ranks (device times must be reduced as the MAX over ranks)."""
    if not dist.is_initialized():
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64,
                     device=device if device is not None else torch.device("cpu"))
    if t.is_cuda:
        t = t.float()
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_counts(count, device=None):
    """sum of an integer over ranks (e.g. frames processed)"""
    if not dist.is_initialized():
        return int(count)
    t = torch.tensor([int(count)], dtype=torch.int64, device=device if device is not None else torch.device("cpu"))
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item())


# --------------------------------------------------------------------------------------------------
# The communication ops below run over torch.distributed (or, for SimSlabGroup, as copies between the ranks' plans).
# While deploy.export records a plan (_lib.recording()), they instead emit the library's collective launch on the
# model file's communicator (occd_comm_*, include/occdepth_b200.h), which the C runtime replays.
class _CommOp:
    def run(self, stream=None):
        if _lib.recording():
            return self._emit(_lib.lib(), stream)
        return self._exchange()


def _nbytes(t):
    return t.numel() * t.element_size()


# X-slab partition of ONE frame across ranks (BASELINE.json configs[2]): the voxel grid is split along X (the
# camera-depth axis; SURVEY.md section 8e explains why not the literal Z), every 3-D activation carries `halo`
# margin planes, and the only data-path communication is the neighbour exchange of those planes before a
# convolution whose taps reach across the slab boundary, plus one all-gather of the CRP mega-context.
def slab_bounds(n, world, stages=0, halo=0, levels=1):
    """X-slab partition of an extent-n axis that a network halves `stages` times: planes [lo, hi) per rank.

    Boundaries are multiples of A = 2**stages, so every rank's slab halves exactly at each stride-2 stage.  Whole
    units of A planes are dealt out as evenly as possible (the first ranks take one more), and a final partial unit
    goes to the last rank.  Every rank must hold at least `halo` planes at each of the first `levels` levels (level k
    has ceil(planes / 2**k) planes), where convolutions reach across the slab boundary.  Where the extent divides
    into world * A planes this is the even split.  Raises SlabPartitionError naming the largest world size that
    works when a rule cannot hold."""
    bounds = _deal(n, world, 1 << stages, halo, levels)
    if bounds is None:
        ok = [r for r in range(world - 1, 0, -1) if _deal(n, r, 1 << stages, halo, levels) is not None]
        raise SlabPartitionError(
            "slab partition: %d X planes in units of %d (%d stride-2 stages) cannot give each of %d ranks at least %d "
            "planes at every exchanging level; the largest world size that works for this grid is %d"
            % (n, 1 << stages, stages, world, halo, ok[0] if ok else 1))
    return bounds


class SlabPartitionError(NotImplementedError):
    pass


def _deal(n, world, unit, halo, levels):
    full, part = divmod(n, unit)
    base, extra = divmod(full, world)
    bounds, lo = [], 0
    for r in range(world):
        hi = lo + (base + (1 if r < extra else 0)) * unit + (part if r == world - 1 else 0)
        bounds.append((lo, hi))
        lo = hi
    if world > 1:
        for k in range(levels):
            if min(level_planes(lo, hi, k) for lo, hi in bounds) < max(halo, 1):
                return None
    if min(hi - lo for lo, hi in bounds) < 1:
        return None
    return bounds


def level_planes(lo, hi, k):
    """planes of the slab [lo, hi) after k stride-2 stages"""
    return -(-hi // (1 << k)) - (lo >> k)


class HaloExchangeOp(_CommOp):
    """Plan op: fill the margins of a halo-carrying activation from the two X-neighbours (send/recv pairs).
    Neighbours may hold different numbers of planes: each side moves min(halo, planes) planes, and the plan only
    exchanges activations every rank holds at least `halo` planes of (Plan.need_halo), so both ends agree."""

    def __init__(self, ctx, cl):
        self.ctx, self.name, self.flops = ctx, "halo_exchange", 0
        buf, h, n = cl.buf, cl.halo, cl.dlen
        w = min(h, n)
        self.bytes = 2 * w * buf[0, 0].numel() * buf.element_size()
        self.send_left, self.recv_left = buf[0, h:h + w], buf[0, h - w:h]
        self.send_right, self.recv_right = buf[0, h + n - w:h + n], buf[0, h + n:h + n + w]
        self.halo, self.planes = h, n
        self._keep = buf

    def _emit(self, L, stream):
        buf = self._keep
        assert buf.shape[0] == 1 and buf.is_contiguous()
        return L.occd_comm_halo_exchange(_lib.MODEL_COMM, buf.data_ptr(), _nbytes(buf[0, 0]), self.halo, self.planes,
                                         stream)

    def _exchange(self):
        c = self.ctx
        ops = []
        if c.rank > 0:
            ops += [dist.P2POp(dist.isend, self.send_left, c.rank - 1), dist.P2POp(dist.irecv, self.recv_left, c.rank - 1)]
        if c.rank < c.world - 1:
            ops += [dist.P2POp(dist.isend, self.send_right, c.rank + 1),
                    dist.P2POp(dist.irecv, self.recv_right, c.rank + 1)]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()


class AllGatherOp(_CommOp):
    """Plan op: dst (full, contiguous) = concat over ranks of src (this rank's contiguous shard).  Shards are equal in
    size; a caller with uneven shards pads each to the largest (CPMegaVoxels.emit)."""

    def __init__(self, ctx, src, dst):
        self.ctx, self.src, self.dst, self.name, self.flops = ctx, src, dst, "all_gather", 0
        self._keep = (src, dst)

    def _emit(self, L, stream):
        assert self.src.is_contiguous() and self.dst.is_contiguous()
        assert _nbytes(self.dst) == self.ctx.world * _nbytes(self.src)
        return L.occd_comm_all_gather(_lib.MODEL_COMM, self.src.data_ptr(), self.dst.data_ptr(), _nbytes(self.src),
                                      stream)

    def _exchange(self):
        dist.all_gather_into_tensor(self.dst, self.src)


class GatherRootOp(_CommOp):
    """Plan op: rank 0 assembles the whole uint16 class map [1, X, Y, Z] from every rank's full-resolution X-slab
    src [1, hi - lo, Y, Z]; bounds[r] = (lo, hi) of rank r.  Rank 0 copies its own slab and receives the others straight
    into their planes of dst (one grouped send/recv); the other ranks send and take dst=None.  The bytes move as uint8,
    whatever the map's element type.  A leading extent of n > 1 gathers n items at once, src [n, hi - lo, Y, Z] into
    dst [n, X, Y, Z] (a map followed by its class probabilities): still one grouped exchange, one send/recv pair per
    item and rank (occd_comm_gather_root_items when recorded)."""

    def __init__(self, ctx, src, dst, bounds):
        self.ctx, self.name, self.flops = ctx, "gather_root", 0
        if not src.is_contiguous() or src.shape[1] != bounds[ctx.rank][1] - bounds[ctx.rank][0]:
            raise RuntimeError("gather_root: rank %d's slab %r does not hold planes %r" % (ctx.rank, tuple(src.shape),
                                                                                       bounds[ctx.rank]))
        self.src, self.dst, self.bounds = src, dst, bounds
        self.parts = None
        if ctx.rank == 0:
            self.parts = [dst[:, lo:hi] for lo, hi in bounds]          # per item contiguous: planes are outermost
        self.bytes = src.numel() * src.element_size()
        self._keep = (src, dst)

    @staticmethod
    def _u8(t):
        return t.reshape(-1).view(torch.uint8)

    def _emit(self, L, stream):
        bounds = (C.c_int * (2 * self.ctx.world))(*[b for lo_hi in self.bounds for b in lo_hi])
        dst = None if self.dst is None else self.dst.data_ptr()
        if self.src.shape[0] > 1:
            return L.occd_comm_gather_root_items(_lib.MODEL_COMM, self.src.data_ptr(), dst, bounds,
                                                 _nbytes(self.src[0, 0]), self.src.shape[0], stream)
        return L.occd_comm_gather_root(_lib.MODEL_COMM, self.src.data_ptr(), dst, bounds, _nbytes(self.src[0, 0]),
                                       stream)

    def _exchange(self):
        c = self.ctx
        items = self.src.shape[0]
        if c.rank == 0:
            self.parts[0].copy_(self.src)
            ops = [dist.P2POp(dist.irecv, self._u8(self.parts[r][i]), r) for r in range(1, c.world)
                   for i in range(items)]
        else:
            ops = [dist.P2POp(dist.isend, self._u8(self.src[i]), 0) for i in range(items)]
        for req in dist.batch_isend_irecv(ops):
            req.wait()


class SlabContext:
    def __init__(self, rank=None, world=None, halo=3):
        w, r, _ = env_world()
        self.rank = r if rank is None else rank
        self.world = w if world is None else world
        self.halo = halo
        self.n_exchanges = 0
        self.bounds = None          # [(lo, hi)] per rank at the lift grid, once partition() has run

    def exchange_op(self, cl):
        self.n_exchanges += 1
        return HaloExchangeOp(self, cl)

    def all_gather_op(self, src, dst):
        return AllGatherOp(self, src, dst)

    def gather_root_op(self, src, dst, bounds):
        return GatherRootOp(self, src, dst, bounds)

    def slab(self, n):
        """planes [lo, hi) of an extent-n axis owned by this rank (n must divide evenly)"""
        if n % self.world:
            raise RuntimeError("slab partition: extent %d is not divisible by %d ranks" % (n, self.world))
        per = n // self.world
        return self.rank * per, (self.rank + 1) * per

    def partition(self, n, stages, levels=3):
        """planes [lo, hi) of the extent-n lift grid owned by this rank under slab_bounds (the 3-D UNets halve X
        `stages` times and exchange halo planes at their first `levels` levels); every rank's bounds are kept for
        the layers that need them (the CRP all-gather)"""
        self.bounds = slab_bounds(n, self.world, stages, self.halo, levels)
        return self.bounds[self.rank]

    def level_bounds(self, extent):
        """every rank's [lo, hi) at the level whose global X extent is `extent`, or None before partition()"""
        if self.bounds is None:
            return None
        n = self.bounds[-1][1]
        for k in range(8):
            if -(-n // (1 << k)) == extent:
                return [(lo >> k, -(-hi // (1 << k))) for lo, hi in self.bounds]
        raise RuntimeError("slab partition: no level of the %d-plane grid has %d planes" % (n, extent))


# --------------------------------------------------------------------------------------------------
# Single-process stand-in for R ranks on ONE device (tests / debugging of the slab partition without R GPUs):
# the R plans are executed in lock-step and the exchange ops copy directly between the plans' buffers.
class SimSlabGroup:
    def __init__(self, world, halo=3):
        self.world, self.ex, self.ag, self.gr = world, {}, {}, {}
        self.ctxs = [SimSlabContext(self, r, world, halo) for r in range(world)]

    @staticmethod
    def run_lockstep(plans, stream=None):
        st = _lib.stream_ptr() if stream is None else stream
        n = len(plans[0].ops)
        assert all(len(p.ops) == n for p in plans), "ranks must build identical op sequences"
        for i in range(n):
            for p in plans:
                p.ops[i].run(st)


class _SimExchangeOp(HaloExchangeOp):
    def __init__(self, ctx, cl, idx):
        super().__init__(ctx, cl)
        self.idx = idx

    def _exchange(self):
        peers = self.ctx.group.ex[self.idx]
        r = self.ctx.rank
        if r > 0:
            self.recv_left.copy_(peers[r - 1].send_right)
        if r < self.ctx.world - 1:
            self.recv_right.copy_(peers[r + 1].send_left)


class _SimAllGatherOp(AllGatherOp):
    def __init__(self, ctx, src, dst, idx):
        super().__init__(ctx, src, dst)
        self.idx = idx

    def _exchange(self):
        peers = self.ctx.group.ag[self.idx]
        flat = self.dst.reshape(self.ctx.world, -1)
        for r in range(self.ctx.world):
            flat[r].copy_(peers[r].src.reshape(-1))


class _SimGatherRootOp(GatherRootOp):
    def __init__(self, ctx, src, dst, bounds, idx):
        super().__init__(ctx, src, dst, bounds)
        self.idx = idx

    def _exchange(self):
        if self.ctx.rank != 0:
            return
        peers = self.ctx.group.gr[self.idx]
        for r in range(self.ctx.world):
            self.parts[r].copy_(peers[r].src)


class SimSlabContext(SlabContext):
    def __init__(self, group, rank, world, halo):
        super().__init__(rank, world, halo)
        self.group, self.n_gathers, self.n_root_gathers = group, 0, 0

    def gather_root_op(self, src, dst, bounds):
        op = _SimGatherRootOp(self, src, dst, bounds, self.n_root_gathers)
        self.group.gr.setdefault(self.n_root_gathers, {})[self.rank] = op
        self.n_root_gathers += 1
        return op

    def exchange_op(self, cl):
        op = _SimExchangeOp(self, cl, self.n_exchanges)
        self.group.ex.setdefault(self.n_exchanges, {})[self.rank] = op
        self.n_exchanges += 1
        return op

    def all_gather_op(self, src, dst):
        op = _SimAllGatherOp(self, src, dst, self.n_gathers)
        self.group.ag.setdefault(self.n_gathers, {})[self.rank] = op
        self.n_gathers += 1
        return op
