"""CPU checks of slab-partition model files (occd_model_load_slab, include/occdepth_b200_comm.h): a well-formed rank
file passes validation on a local communicator; occd_model_load, the communicator's rank and world, a communicator
argument in a plain file, bounds that do not tile the grid, the index window and the staged view are refused with
their code and message before any device is touched; an unloadable NCCL is OCCD_ERR_UNSUPPORTED; the collective
launches refuse a NULL communicator; and the recording of each communication op of parallel.SimSlabContext is a
record the runtime's table accepts."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib, deploy
from occdepth_b200.engine import CL
from occdepth_b200.parallel import SimSlabGroup


def _lib_built():
    _build.build()
    return _lib.lib()


def _arg(tag, *v):
    fmt = {"p": "<IQ", "h": "<I", "c": "<I", "i": "<i", "l": "<q", "f": "<f", "d": "<d", "n": "", "s": "", "m": ""}[tag]
    return tag.encode() + (struct.pack(fmt, *v) if fmt else b"")


def _record(name, args):
    nm = name.encode()
    return struct.pack("<H", len(nm)) + nm + struct.pack("<I", len(args)) + b"".join(args)


GATHER = _record("occd_comm_all_gather", [_arg("m"), _arg("p", 0, 0), _arg("p", 0, 64), _arg("l", 8), _arg("s")])


def slab_file(rank=0, world=2, bounds=None, window=None, view_sel=-1, map_x=2, slab=True, records=(GATHER,),
              blobs=(), extra=()):
    """rank `rank` of a tiny model split over `world` ranks: one 2 x 2 image, a 2 x 1 x 2 grid (X planes split by
    `bounds`), one buffer per staged role (the class map on rank 0 only), then the buffers `extra`"""
    bounds = bounds or [(0, 1), (1, 2)]
    plane = 1 * 2
    lo, hi = bounds[rank] if rank < len(bounds) else (0, 1)
    n_lo, n_len = window or (lo * plane, (hi - lo) * plane)
    n = n_len if slab else 2 * plane
    roles_len = [2 * 2 * 8 * 4, n * 16, n, n * 8, 0, 0, 0, 2 * 2 * 2 if rank == 0 else 0]
    bufs = [k for k in roles_len if k] + list(extra)
    roles, k = [], 0
    for ln in roles_len:
        roles.append((k, 0, ln) if ln else (-1, 0, 0))
        k += 1 if ln else 0
    abi = _lib_built().occd_abi_version()
    hdr = deploy.MAGIC + struct.pack("<9I", _lib.MODEL_FORMAT_VERSION, abi, 0, 0, deploy.FLAG_SLAB if slab else 0,
                                     1, 2, 2, 1)
    hdr += struct.pack("<7I", 2, 1, 2, 2, 1, 2, 1)
    hdr += np.zeros(128, "<i4").tobytes() + struct.pack("<7d", 0.4, 0, 0, 0, 0.8, 0.4, 0.8)
    hdr += struct.pack("<2I", 20, 0) + np.zeros(64, "<i4").tobytes() + struct.pack("<d3I", 0.0, 0, 0, 0)
    hdr += struct.pack("<3I", 0, 0, 0) + np.zeros(16, "<f4").tobytes() + struct.pack("<I", 8)
    hdr += b"".join(struct.pack("<iQQ", *r) for r in roles)
    if slab:
        hdr += struct.pack("<2I", rank, world) + b"".join(struct.pack("<2I", *b) for b in bounds)
        hdr += struct.pack("<2QiI", n_lo, n_len, view_sel, map_x)
    hdr += struct.pack("<4I", len(bufs), len(blobs), 0, len(records))
    body = b"".join(struct.pack("<QI", ln, 0) for ln in bufs)
    for data, fix in blobs:
        body += struct.pack("<Q", len(data)) + data + struct.pack("<I", len(fix))
        body += b"".join(struct.pack("<QIQ", *f) for f in fix)
    return hdr + body + b"".join(records)


def _local(world):
    hs = (C.c_void_p * world)()
    assert _lib_built().occd_comm_create_local(world, hs) == 0
    return [C.c_void_p(h) for h in hs]


def _load(tmp_path, data, comm=None):
    L = _lib_built()
    p = tmp_path / "m.occd"
    p.write_bytes(data)
    h = C.c_void_p()
    rc = (L.occd_model_load(str(p).encode(), C.byref(h)) if comm is None
          else L.occd_model_load_slab(str(p).encode(), comm, C.byref(h)))
    if rc == 0:
        L.occd_model_destroy(h)
    else:
        assert not h.value
    return rc, L.occd_last_error().decode()


def _passes_validation(rc, msg):
    """a valid file either loads (a GPU is present) or stops at the first CUDA call"""
    return rc == 0 or (rc == _lib.ERR_CUDA and "cudaMalloc" in msg)


def _destroy(comms):
    for c in comms:
        _lib.lib().occd_comm_destroy(c)


@pytest.mark.parametrize("rank", [0, 1])
def test_well_formed_slab_file_passes_validation(tmp_path, rank):
    comms = _local(2)
    try:
        rc, msg = _load(tmp_path, slab_file(rank=rank), comms[rank])
        assert _passes_validation(rc, msg), (rc, msg)
        # a NULL communicator slot passes the loader (the launch refuses it when it runs)
        null_comm = _record("occd_comm_all_gather", [_arg("n"), _arg("p", 0, 0), _arg("p", 0, 64), _arg("l", 8),
                                                     _arg("s")])
        rc, msg = _load(tmp_path, slab_file(rank=rank, records=[null_comm]), comms[rank])
        assert _passes_validation(rc, msg), (rc, msg)
    finally:
        _destroy(comms)


@pytest.mark.parametrize("case,code,text", [
    ("plain_loader", _lib.ERR_UNSUPPORTED, "load it with occd_model_load_slab"),
    ("rank", _lib.ERR_ARG, "the file is rank 1 of 2, the communicator rank 0 of 2"),
    ("world", _lib.ERR_ARG, "the file is rank 0 of 2, the communicator rank 0 of 3"),
    ("comm_in_plain_file", _lib.ERR_FORMAT, "a communicator in a file without the slab partition"),
    ("plain_file_slab_loader", _lib.ERR_UNSUPPORTED, "holds no X-slab partition"),
    ("bounds_gap", _lib.ERR_FORMAT, "do not tile the 2 X planes"),
    ("bounds_short", _lib.ERR_FORMAT, "do not tile the 2 X planes"),
    ("bounds_start", _lib.ERR_FORMAT, "do not tile the 2 X planes"),
    ("window", _lib.ERR_FORMAT, "index window"),
    ("view_sel", _lib.ERR_FORMAT, "staged view 1 outside [-1, 1)"),
    ("view_sel_neg", _lib.ERR_FORMAT, "staged view -2 outside"),
    ("map_x", _lib.ERR_FORMAT, "map extent"),
    ("world_range", _lib.ERR_FORMAT, "out of range"),
])
def test_slab_loader_refuses(tmp_path, case, code, text):
    comms2, comms3 = _local(2), _local(3)
    try:
        comm = {"world": comms3[0], "rank": comms2[0], "plain_loader": None,
                "comm_in_plain_file": None}.get(case, comms2[0])
        data = {
            "plain_loader": lambda: slab_file(),
            "rank": lambda: slab_file(rank=1),
            "world": lambda: slab_file(),
            "comm_in_plain_file": lambda: slab_file(slab=False),
            "plain_file_slab_loader": lambda: slab_file(slab=False, records=()),
            "bounds_gap": lambda: slab_file(bounds=[(0, 1), (2, 2)]),
            "bounds_short": lambda: slab_file(bounds=[(0, 1), (1, 1)]),
            "bounds_start": lambda: slab_file(bounds=[(1, 1), (1, 2)]),
            "window": lambda: slab_file(window=(2, 2)),
            "view_sel": lambda: slab_file(view_sel=1),
            "view_sel_neg": lambda: slab_file(view_sel=-2),
            "map_x": lambda: slab_file(map_x=4),
            "world_range": lambda: slab_file(world=65),
        }[case]()
        rc, msg = _load(tmp_path, data, comm)
        assert rc == code, (rc, msg)
        assert text in msg, msg
    finally:
        _destroy(comms2 + comms3)


def test_unloadable_nccl_is_unsupported(tmp_path):
    L = _lib_built()
    bad = str(tmp_path / "no" / "libnccl.so.2").encode()
    buf = C.create_string_buffer(_lib.COMM_ID_BYTES)
    assert L.occd_comm_unique_id(bad, buf) == _lib.ERR_UNSUPPORTED
    assert b"cannot load NCCL" in L.occd_last_error()
    h = C.c_void_p()
    assert L.occd_comm_create(bad, buf, 0, 2, C.byref(h)) == _lib.ERR_UNSUPPORTED and not h.value
    assert b"cannot load NCCL" in L.occd_last_error()
    assert L.occd_comm_create(bad, buf, 2, 2, C.byref(h)) == _lib.ERR_ARG          # rank checked first
    with pytest.raises(RuntimeError, match="cannot load NCCL"):
        deploy.Comm.unique_id(tmp_path / "no" / "libnccl.so.2")


def test_collectives_refuse_a_null_communicator():
    L = _lib_built()
    b = (C.c_int * 4)(0, 1, 1, 2)
    for rc in (L.occd_comm_halo_exchange(None, 1, 8, 1, 1, None), L.occd_comm_all_gather(None, 1, 1, 8, None),
               L.occd_comm_gather_root(None, 1, 1, b, 8, None)):
        assert rc == _lib.ERR_ARG
        assert b"no communicator" in L.occd_last_error()


def test_recorded_collective_ops_are_replayable(tmp_path):
    """parallel's communication ops, recorded as deploy.export records them (without running), on both ranks of a
    SimSlabGroup: each becomes a record of its occd_comm_* launch on the model's communicator ('m') that the runtime's
    table accepts; the simulated copies do not run"""
    grp = SimSlabGroup(2, halo=1)
    arena = torch.zeros(4096, dtype=torch.uint8)                    # stands in for one device buffer
    base = arena.data_ptr()
    for r, ctx in enumerate(grp.ctxs):
        act = arena[:2 * 4 * 8 * 4].view(torch.float32).view(1, 4, 1, 2, 8)      # 2 planes + 1 halo on each side
        act.fill_(1.0)
        src = arena[1024:1032].view(torch.uint16).view(1, 1, 2, 2)               # one plane of the class map
        dst = arena[2048:2064].view(torch.uint16).view(1, 2, 2, 2)
        ops = [ctx.exchange_op(CL(act, 8, 0, 1, 2)), ctx.all_gather_op(arena[3072:3080], arena[3200:3216]),
               ctx.gather_root_op(src, dst if r == 0 else None, [(0, 1), (1, 2)])]
        rec = deploy._Recorder(_lib_built())
        rec.recording = True
        _lib._RECORDING.recorder = rec
        try:
            for op in ops:
                op.run(deploy._STREAM)
        finally:
            _lib._RECORDING.recorder = None
        assert [c[0] for c in rec.calls] == ["occd_comm_halo_exchange", "occd_comm_all_gather",
                                             "occd_comm_gather_root"]
        assert all(c[1][0] == ("m",) and c[1][-1] == ("s",) for c in rec.calls)
        assert rec.calls[0][1][2:5] == [("l", 2 * 8 * 4), ("i", 1), ("i", 2)]
        assert rec.calls[1][1][3] == ("l", 8)
        assert rec.calls[2][1][4] == ("l", 2 * 2 * 2)
        assert not dst.any() and not arena[3200:3216].any()               # nothing ran
        # the arena is the buffer after the roles' (rank 0: img pix fov pix_z classes; rank 1: no class map)
        arena_id = 5 if r == 0 else 4
        records, blobs = [], []
        for name, args in rec.calls:
            enc = []
            for a in args:
                if a[0] == "p":
                    enc.append(_arg("p", arena_id, a[1] - base))
                elif a[0] == "h":
                    blobs.append((a[1][0], []))
                    enc.append(_arg("h", len(blobs) - 1))
                else:
                    enc.append(_arg(*a))
            records.append(_record(name, enc))
        comms = _local(2)
        try:
            rc, msg = _load(tmp_path, slab_file(rank=r, records=records, blobs=blobs, extra=[4096]), comms[r])
            assert _passes_validation(rc, msg), (r, rc, msg)
        finally:
            _destroy(comms)
