"""Python-free deployment: export a model's camera-frame class-map plan to one self-contained model file, which
libocc_b200.so loads and replays from C (`occd_model_load` / `occd_model_run_frame`, include/occdepth_b200.h;
tools/occd_run.c is a standalone consumer).  The file layout is documented in DESIGN.md section 9.

The export records, it does not re-describe: the plan is built by the same `OccDepth._build` that
`predict_frame` uses, while `_lib.lib()` returns a recording stand-in, and then run once through it.  Every call the
run makes becomes a record (entry point name + arguments typed by `_lib.SYMBOLS`); device pointers become
(buffer, offset) pairs into the storages the plan holds, host structs and arrays become byte blobs with pointer
fix-ups, and convolution plans are stored as the descriptors they were created from.  No model code knows about
export, so a launch a model adds later is exported as it is.
"""
import bisect
import ctypes as C
import os
import struct

import numpy as np
import torch

from . import _lib
from .engine import CL, ConvOp

MAGIC = b"OCCDMODL"
ROLES = ("img", "pix", "fov", "pix_z", "depth", "cams", "sps", "classes")
FLAG_FLOSP_DEPTH, FLAG_VIRTUAL, FLAG_CONF, FLAG_SLAB = 1, 2, 4, 16  # FLAG_CONF: the class-map role holds the map,
                                                                   # then its float16 confidence; FLAG_SLAB: one
                                                                   # rank's plan of the X-slab partition
FLAG_BATCH = 32                                                    # a B-frame plan of predict_frames (batch block)
FLAG_MAPS = 64                                                     # the staged views' rectification maps (maps role)
PATTERN_MAX = 64

_STREAM = object()        # the launch stream of the recording run: becomes the stream slot of a record
# forwarded even while recording: queries, and the destructors -- a ConvOp or LoadedModel of another plan that the
# garbage collector finalizes on the exporting thread during the recording run is released, not recorded
_PASS_THROUGH = {"occd_last_error", "occd_abi_version", "occd_conv_plan_info", "occd_conv_plan_impl",
                 "occd_conv_plan_schedule", "occd_conv_plan_destroy", "occd_model_destroy"}


class ExportError(RuntimeError):
    """the plan holds something a model file cannot carry (a pointer outside every buffer the plan holds, an
    argument of unknown kind)"""


def _ptr_offsets(t, base=0):
    """byte offsets of the c_void_p fields of ctypes type `t` (structs and arrays, recursively)"""
    if t is C.c_void_p:
        return [base]
    if isinstance(t, type) and issubclass(t, C.Array):
        step = C.sizeof(t._type_)
        return [o for i in range(t._length_) for o in _ptr_offsets(t._type_, base + i * step)]
    if isinstance(t, type) and issubclass(t, C.Structure):
        return [o for f in t._fields_ for o in _ptr_offsets(f[1], base + getattr(t, f[0]).offset)]
    return []


def _host_blob(obj):
    """ctypes object -> (bytes, [(offset, pointer value)]) of its host memory and the device pointers inside it"""
    raw = bytearray(C.string_at(C.addressof(obj), C.sizeof(obj)))
    ptrs = []
    for off in _ptr_offsets(type(obj)):
        v = int.from_bytes(raw[off:off + 8], "little")
        if v:
            ptrs.append((off, v))
            raw[off:off + 8] = bytes(8)
    return bytes(raw), ptrs


class _Recorder:
    """stands in for the loaded library: forwards every call while the plan is built (recording the convolution
    plans created and their class LUTs), then records without executing while the plan runs"""

    def __init__(self, real):
        self._real = real
        self.recording = False
        self.plans = {}            # handle value -> [descriptor blob, (lut bytes, n) or None]
        self.calls = []            # (entry point, [raw argument])

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name not in _lib.SYMBOLS:
            return fn
        argtypes = _lib.SYMBOLS[name][1]

        def call(*args):
            if not self.recording or name in _PASS_THROUGH:
                rc = fn(*args)
                if rc == 0 and name == "occd_conv_plan_create":
                    self.plans[args[1]._obj.value] = [_host_blob(args[0]._obj), None]
                elif rc == 0 and name == "occd_conv_plan_set_class_lut":
                    lut = None if args[1] is None else (bytes(args[1]), int(args[2]))
                    self.plans[_handle(args[0])][1] = lut
                return rc
            self.calls.append((name, [self._arg(name, i, a, t) for i, (a, t) in enumerate(zip(args, argtypes))]))
            return 0
        return call

    def _arg(self, name, i, a, t):
        if t is C.c_int or t is C.c_longlong:
            return ("i" if t is C.c_int else "l", int(getattr(a, "value", a)))
        if t is C.c_float or t is C.c_double:
            return ("f" if t is C.c_float else "d", float(getattr(a, "value", a)))
        if a is _STREAM:
            return ("s",)
        if a is _lib.MODEL_COMM:
            return ("m",)
        if name == "occd_conv_run" and i == 0:
            h = _handle(a)
            if h not in self.plans:
                raise ExportError("export: occd_conv_run argument 0: a convolution plan created outside the build")
            return ("c", h)
        if a is None:
            return ("n",)
        if type(a).__name__ == "CArgObject":               # C.byref(struct)
            return ("h", _host_blob(a._obj))
        if isinstance(a, (C.Array, C.Structure)):
            return ("h", _host_blob(a))
        v = a.value if isinstance(a, C.c_void_p) else a
        if v is None or (isinstance(v, (int, np.integer)) and int(v) == 0):
            return ("n",)
        if isinstance(v, (int, np.integer)):
            return ("p", int(v))
        raise ExportError("export: %s argument %d: cannot record a %s" % (name, i, type(a).__name__))


def _handle(h):
    return h.value if isinstance(h, C.c_void_p) else int(h)


def _collect(obj, out):
    if isinstance(obj, torch.Tensor):
        out.append(obj)
    elif isinstance(obj, CL):
        out.append(obj.buf)
    elif isinstance(obj, (list, tuple)):
        for x in obj:
            _collect(x, out)
    elif isinstance(obj, dict):
        for x in obj.values():
            _collect(x, out)


class _Buffers:
    """the device storages a plan holds, overlapping ones merged, with their contents"""

    def __init__(self, tensors):
        spans = {}
        for t in tensors:
            if t.is_cuda:
                s = t.untyped_storage()
                spans[s.data_ptr()] = s
        iv = []                                         # [base, end, [storages]]
        for base in sorted(spans):
            s = spans[base]
            end = base + s.nbytes()
            if iv and base < iv[-1][1]:
                iv[-1][1] = max(iv[-1][1], end)
                iv[-1][2].append(s)
            else:
                iv.append([base, end, [s]])
        self.iv = iv
        self.bases = [b for b, _, _ in iv]

    def place(self, p, what):
        k = bisect.bisect_right(self.bases, p) - 1
        if k < 0 or not p < self.iv[k][1]:
            raise ExportError("export: %s: pointer 0x%x lands in no buffer the plan holds" % (what, p))
        return k, p - self.iv[k][0]

    def contents(self, k):
        """bytes of buffer k, or None when it is all zeros"""
        base, end, storages = self.iv[k]
        out = np.zeros(end - base, dtype=np.uint8)
        for s in storages:
            u8 = torch.empty(0, dtype=torch.uint8, device=s.device).set_(s, 0, (s.nbytes(),), (1,))
            o = s.data_ptr() - base
            out[o:o + s.nbytes()] = u8.cpu().numpy()
        return out.tobytes() if out.any() else None


def export(model, path, frame, inv_map=None, confidence=False, slab_output=None):
    """Write the model file of `model.predict_frame(frame, classes=True, inv_map=inv_map, confidence=confidence)`
    for frames of this frame's shape (image count and size, depth map size, voxel grid).  Refuses what predict_frame
    refuses, with the same messages.  Returns a dict of what was written (records, buffers, bytes).

    `frame` a list of B frames: the file of `model.predict_frames(frame, ...)`, B frames per run (header flag
    FLAG_BATCH and a batch block; every role holds B items), which `occd_model_run_frames` replays for 1..B frames.
    Refuses what predict_frames refuses; not with slab_output.  With
    `confidence` the file's class-map role holds the map and then its confidence (header flag FLAG_CONF), which
    `occd_model_run_frame_conf` reads; without it the file is what it always was.

    A frame carrying "rect_maps" embeds them (header flag FLAG_MAPS and a maps role after the roles): a rig's
    calibration is fixed per deployment, so the runtime rectifies every frame with them (a slab file holds its staged
    view's only).  The frames of a batched export must then all carry the same maps.  Neither the frame's pixel
    format nor its maps change the plan; the format is the caller's per run (`occd_model_run_frames_ex`).

    Under enable_slab_parallel, slab_output="root" (the only value a file carries) writes this rank's plan of
    `predict_frame(frame, slab_output="root", ...)`: every rank exports the same frame to its own path, and the
    files are loaded by `occd_model_load_slab` on each rank's communicator (header flag FLAG_SLAB and a slab block).
    The recording runs no collective: the plan's communication ops emit the library's collective launches instead,
    so the ranks' plans may also be built one after another on one device (parallel.SimSlabGroup contexts).

    The recording stand-in replaces the library for the calling thread only, so other threads may keep serving
    through the library meanwhile; `model` itself must not run elsewhere during the export (as for predict_frame)."""
    from . import data as D
    batched = not isinstance(frame, dict)
    if batched:
        if slab_output is not None:
            raise NotImplementedError("deploy.export: a batched model file (a list of frames) has no X-slab partition")
        fs = model._frames_checked(frame, True, confidence)
        f, B = fs[0], len(frame)
        for i, fi in enumerate(fs[1:], 1):
            if (fi["maps"] is None) != (f["maps"] is None) or (fi["maps"] is not None
                                                              and not torch.equal(fi["maps"], f["maps"])):
                raise ValueError("deploy.export: frame %d's rect_maps differ from frame 0's; a model file holds one "
                                 "set of maps for every frame" % i)
    else:
        f = model._frame_checked(frame, slab_output)
        B = 1
    depth_items = f["virtual"] and B > 1
    slab = model.__dict__.get("slab_ctx")
    if slab_output == "slab":
        raise NotImplementedError("deploy.export: a model file holds the whole map on rank 0 (slab_output='root'); "
                                  "per-rank slabs are not exported")
    lut = model._class_lut(inv_map)
    dev = f["imgs"].device
    rec = _Recorder(_lib.lib())
    with torch.cuda.device(dev), torch.no_grad():
        _lib._RECORDING.recorder = rec
        try:
            ent = model._build(B, f["V"], f["H"], f["W"], f["N"], f["P"], dev, f["batch"],
                               classes=model._class_key(inv_map, confidence, slab is not None), capture=False,
                               depth_items=depth_items)
            plan, img_cl, pix, fov, out, depth0, n_lo, view_sel = ent
            plan.pix_z = torch.zeros(pix.shape[0], pix.shape[2], dtype=torch.float64, device=dev)
            state = getattr(plan, "flosp_state", None)
            tensors = []
            for op in plan.ops:
                _collect(getattr(op, "_keep", ()), tensors)
                if isinstance(op, ConvOp):
                    tensors += [op.weight, op.bias]
            maps = None
            if f["maps"] is not None:         # the staged views' maps, in a buffer of their own
                maps = (f["maps"] if view_sel is None else f["maps"][view_sel:view_sel + 1]).contiguous().clone()
            _collect([img_cl, pix, fov, out, depth0, plan.pix_z, state, maps], tensors)
            torch.cuda.synchronize()
            bufs = _Buffers(tensors)
            contents = [bufs.contents(k) for k in range(len(bufs.iv))]     # before the run: activations are zero
            rec.recording = True
            plan.run(_STREAM)
        finally:
            rec.recording = False
            _lib._RECORDING.recorder = None

    blobs, plan_ids = [], {}

    def blob(b, what):
        data, ptrs = b
        blobs.append((data, [(o,) + bufs.place(v, what) for o, v in ptrs]))
        return len(blobs) - 1

    records = []
    for name, args in rec.calls:
        enc = []
        for i, a in enumerate(args):
            what = "%s argument %d" % (name, i)
            if a[0] == "p":
                enc.append(("p",) + bufs.place(a[1], what))
            elif a[0] == "h":
                enc.append(("h", blob(a[1], what)))
            elif a[0] == "c":
                if a[1] not in plan_ids:
                    plan_ids[a[1]] = len(plan_ids)
                enc.append(("c", plan_ids[a[1]]))
            else:
                enc.append(a)
        records.append((name, enc))
    plans = []
    for h, pid in sorted(plan_ids.items(), key=lambda kv: kv[1]):
        desc, lut_rec = rec.plans[h]
        d = blob(desc, "occd_conv_plan_create descriptor")
        if lut_rec is None:
            plans.append((d, -1, 0))
        else:
            blobs.append((lut_rec[0], []))
            plans.append((d, len(blobs) - 1, lut_rec[1]))

    def role(t):
        if t is None:
            return (-1, 0, 0)
        assert t.is_contiguous()
        k, off = bufs.place(t.data_ptr(), "role buffer")
        return (k, off, t.numel() * t.element_size())

    roles = [role(img_cl.buf), role(pix), role(fov), role(plan.pix_z), role(depth0),
             role(state["cams"] if state else None), role(state["sps"] if state else None), role(out)]
    flosp = model.trans_2d_to_3d == "flosp_depth"
    nyu = model.dataset == "NYU"
    G = np.zeros(16, np.float32)
    n_cams, vn = 0, (0, 0, 0)
    if flosp:
        n_cams, vn = int(state["n_cams"]), tuple(int(v) for v in state["vn"])
        if not nyu:
            G = model.flosp_depth._grid_to_lidar(None)[0].numpy().reshape(-1)
    pattern = np.zeros((PATTERN_MAX, 2), np.int32)
    pattern[:f["P"]] = np.asarray(D.PIXEL_PATTERNS[f["pattern_id"]], np.int32)
    lut_arr = np.zeros(_lib.CLASS_LUT_MAX, np.int32)
    if lut is not None:
        lut_arr[:len(lut)] = lut
    S = [int(s) // model.project_scale for s in model.full_scene_size]
    # the whole map on every rank's header (rank 0's output; the other ranks' plans output nothing)
    out_dims = tuple(out.shape[-3:]) if out is not None else tuple(int(s) for s in model.full_scene_size)
    hdr = [MAGIC, struct.pack("<9I", _lib.MODEL_FORMAT_VERSION, _lib.lib().occd_abi_version(), plan.lib_dtype,
                              1 if nyu else 0, (FLAG_FLOSP_DEPTH if flosp else 0) | (FLAG_VIRTUAL if f["virtual"] else 0)
                              | (FLAG_CONF if confidence else 0) | (FLAG_SLAB if slab is not None else 0)
                              | (FLAG_BATCH if batched else 0) | (FLAG_MAPS if maps is not None else 0),
                              f["V"], f["H"], f["W"], model.project_scale),
           struct.pack("<7I", *S, *out_dims, f["P"]), pattern.astype("<i4").tobytes(),
           struct.pack("<7d", float(f["voxel_size"]), *[float(v) for v in f["vox_origin"]],
                       *[float(v) for v in f["scene_size"]]),
           struct.pack("<2I", model.n_classes, 0 if lut is None else 1), lut_arr.astype("<i4").tobytes(),
           struct.pack("<d3I", float(f["virtual_bf"]), *(depth0.shape[-2:] if depth0 is not None else (0, 0)), n_cams),
           struct.pack("<3I", *vn),
           G.astype("<f4").tobytes(), struct.pack("<I", img_cl.cstride)]
    hdr += [struct.pack("<iQQ", *r) for r in roles]
    if maps is not None:
        hdr.append(struct.pack("<iQQ", *role(maps)))
    if batched:
        hdr.append(struct.pack("<I", B))
    if slab is not None:
        # rank, world, every rank's [lo, hi) of the lift grid, this rank's index window, its staged view, the whole
        # map's X extent
        hdr.append(struct.pack("<2I", slab.rank, slab.world)
                   + struct.pack("<%dI" % (2 * slab.world), *[b for lo_hi in slab.bounds for b in lo_hi])
                   + struct.pack("<2QiI", n_lo, pix.shape[2], -1 if view_sel is None else view_sel, out_dims[0]))
    hdr.append(struct.pack("<4I", len(bufs.iv), len(blobs), len(plans), len(records)))
    n_bytes = 0
    with open(path, "wb") as fh:
        def w(b):
            nonlocal n_bytes
            fh.write(b)
            n_bytes += len(b)
        for b in hdr:
            w(b)
        for k, (base, end, _) in enumerate(bufs.iv):
            w(struct.pack("<QI", end - base, 0 if contents[k] is None else 1))
            if contents[k] is not None:
                w(contents[k])
        for data, fix in blobs:
            w(struct.pack("<Q", len(data)) + data + struct.pack("<I", len(fix)))
            for o, k, off in fix:
                w(struct.pack("<QIQ", o, k, off))
        for p in plans:
            w(struct.pack("<IiI", *p))
        for name, enc in records:
            nm = name.encode()
            w(struct.pack("<H", len(nm)) + nm + struct.pack("<I", len(enc)))
            for a in enc:
                tag = a[0].encode()
                if a[0] == "p":
                    w(tag + struct.pack("<IQ", a[1], a[2]))
                elif a[0] in "hc":
                    w(tag + struct.pack("<I", a[1]))
                elif a[0] in "ilfd":
                    w(tag + struct.pack("<" + {"i": "i", "l": "q", "f": "f", "d": "d"}[a[0]], a[1]))
                else:
                    w(tag)
    return dict(records=len(records), buffers=len(bufs.iv), plans=len(plans), bytes=n_bytes,
                data_buffers=sum(c is not None for c in contents))


class Comm:
    """a communicator of the library (occd_comm, include/occdepth_b200_comm.h) for slab-partition model files.
    Comm(id, rank, world): NCCL, one rank per process on the current device, collective over the ranks; `id` is
    Comm.unique_id() of rank 0, shipped to the others by the caller.  Comm.local(world): `world` ranks in this process
    on the current device, run together by run_frame_group.  `nccl_lib`: the path of libnccl.so.2 (None: the soname,
    which torch has usually loaded already)."""

    def __init__(self, id=None, rank=0, world=1, nccl_lib=None, _handle=None):
        self.rank, self.world = rank, world
        if _handle is not None:
            self.handle = _handle
            return
        h = C.c_void_p()
        _lib.check(_lib.lib().occd_comm_create(_path(nccl_lib), bytes(id), rank, world, C.byref(h)),
                   "occd_comm_create")
        self.handle = h

    @staticmethod
    def unique_id(nccl_lib=None):
        buf = C.create_string_buffer(_lib.COMM_ID_BYTES)
        _lib.check(_lib.lib().occd_comm_unique_id(_path(nccl_lib), buf), "occd_comm_unique_id")
        return buf.raw

    @classmethod
    def local(cls, world):
        hs = (C.c_void_p * world)()
        _lib.check(_lib.lib().occd_comm_create_local(world, hs), "occd_comm_create_local")
        return [cls(rank=r, world=world, _handle=C.c_void_p(hs[r])) for r in range(world)]

    def close(self):
        if self.handle:
            _lib.lib().occd_comm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def _path(p):
    return None if p is None else os.fsencode(p)


class LoadedModel:
    """ctypes handle of a model file loaded by the C runtime (occd_model_load), for Python callers that want the
    Python-free route's results: `run_frame` takes the frame dict of OccDepth.predict_frame.  With `comm` (a Comm)
    the file is one rank's of the X-slab partition (occd_model_load_slab); the model keeps the communicator alive."""

    def __init__(self, path, comm=None):
        L = _lib.lib()
        h = C.c_void_p()
        if comm is None:
            _lib.check(L.occd_model_load(os.fsencode(path), C.byref(h)), "occd_model_load(%s)" % path)
        else:
            _lib.check(L.occd_model_load_slab(os.fsencode(path), comm.handle, C.byref(h)),
                       "occd_model_load_slab(%s)" % path)
        self.handle = h
        self.comm = comm
        self.geom = self.info()
        self._last_n = 0               # frames of the last run through this object (list_voxels' default n)

    def info(self):
        g = _lib.ModelGeom()
        _lib.check(_lib.lib().occd_model_info(self.handle, C.byref(g)), "occd_model_info")
        return g

    def batch(self):
        """frames per run: B of a file exported from a list of frames, 1 otherwise"""
        b = C.c_int()
        _lib.check(_lib.lib().occd_model_batch(self.handle, C.byref(b)), "occd_model_batch")
        return b.value

    def run_frames(self, frames, out=None, stream=None, graph=True, conf=None, pixel_format=None):
        """1..B frames (as OccDepth.predict_frames takes them) through occd_model_run_frames -> uint16 [n, X, Y, Z] on
        the current device, or (map, conf) with `conf` (a float16 [n, X, Y, Z] device tensor, or True).
        Each frame's "pixel_format" ("rgb" by default, "bgr", or "nv12": then its "img" is uint8 (V, H0 * 3 / 2, W0),
        OpenCV's NV12 layout) is staged through occd_model_run_frames_ex; `pixel_format` sets it for every frame, and a
        frame whose own key says otherwise is refused.  The file's rectification maps apply: a frame carrying
        "rect_maps" is refused."""
        n = len(frames)
        if pixel_format is not None and pixel_format not in _lib.PIXEL_FORMATS:
            raise ValueError("LoadedModel.run_frames: pixel_format must be 'rgb', 'bgr' or 'nv12', got %r"
                             % (pixel_format,))
        fmts = [pixel_format or fr.get("pixel_format", "rgb") for fr in frames]
        calls = [_frame_call(self.geom, fr, None, None, graph, None, False, fmt, "LoadedModel.run_frames")
                 for fr, fmt in zip(frames, fmts)]
        if all(fmt == "rgb" for fmt in fmts):
            fa = (_lib.Frame * n)(*[c[0] for c in calls])
            run = _lib.lib().occd_model_run_frames
        else:
            fa = (_lib.FrameEx * n)(*[_lib.FrameEx(c[0], _lib.PIXEL_FORMATS[fmt], c[1][0].stride(1) * c[0].H0)
                                      for c, fmt in zip(calls, fmts)])
            run = _lib.lib().occd_model_run_frames_ex
        dev = calls[0][1][0].device                 # the first frame's images, on the device
        if out is None:
            out = torch.empty(n, self.geom.X, self.geom.Y, self.geom.Z, dtype=torch.uint16, device=dev)
        if conf is True:
            conf = torch.empty(out.shape, dtype=torch.float16, device=dev)
        assert out.dtype == torch.uint16 and out.is_contiguous() and out.shape[0] == n
        if conf is not None:
            assert conf.dtype == torch.float16 and conf.is_contiguous() and conf.shape == out.shape
        keep = [c[1] for c in calls]
        st = _stream_for(stream, [t for c in keep for t in c if isinstance(t, torch.Tensor)] + [out, conf])
        self._last_n = 0
        _lib.check(run(self.handle, fa, n, _ptr(out), _ptr(conf), st), run.__name__)
        self._last_n = n
        return out if conf is None else (out, conf)

    def run_frame(self, frame, out=None, stream=None, graph=True, conf=None):
        """frame: as OccDepth.predict_frame takes it (the uint8 images may be on the host or the device) -> the
        uint16 class map [1, X, Y, Z] on the current device, enqueued on `stream` (default: the current stream).
        `conf`: a float16 [1, X, Y, Z] device tensor (or True: allocate one) that gets the map's confidence through
        occd_model_run_frame_conf; the result is then (map, conf).  On a slab rank other than 0 nothing is written
        and the result is None; every rank must run every frame (with conf on every rank or on none)."""
        root = self.comm is None or self.comm.rank == 0
        f, keep, out, conf_t, st = _frame_call(self.geom, frame, out, stream, graph, conf, root, "rgb",
                                               "LoadedModel.run_frame")
        self._last_n = 0
        if conf is None:
            _lib.check(_lib.lib().occd_model_run_frame(self.handle, C.byref(f), _ptr(out), st), "occd_model_run_frame")
            self._last_n = 1
            return out if root else None
        _lib.check(_lib.lib().occd_model_run_frame_conf(self.handle, C.byref(f), _ptr(out), _ptr(conf_t), st),
                   "occd_model_run_frame_conf")
        self._last_n = 1
        return (out, conf_t) if root else None

    def list_voxels(self, n=None, capacity=None, voxel_size=None, vox_origin=None, xyz=True, out=None, stream=None):
        """The occupied-voxel list of the maps the last run left on the device (occd_model_list_voxels) ->
        voxels.VoxelList with B = n, enqueued on `stream` (default: the current stream); nothing is read back until
        the caller asks the list for counts or rows.  Bit for bit OccDepth.predict_voxels of the frames that run saw:
        rows split by each frame's fov_mask_1 (KITTI; NYU lists every row as inside), labels remapped when the file
        was exported with inv_map.  Works after run_frame, run_frames and run_frame_group (on models[0]).

        n: items [0, n) of the last run (default: all of them).  capacity: rows per frame (default N: never
        truncates).  voxel_size: of the output grid (default 0.2 KITTI, 0.08 NYU); vox_origin: added to the centres;
        xyz=False: no coordinates.  out: a VoxelList of an earlier call with the same n, capacity and xyz, whose
        tensors are overwritten."""
        from .voxels import VoxelList
        g = self.geom
        n = self._last_n if n is None else int(n)
        N = g.X * g.Y * g.Z
        cap = N if capacity is None else int(capacity)
        if cap < 0:
            raise ValueError("LoadedModel.list_voxels: capacity must be >= 0")
        if vox_origin is not None and not xyz:
            raise ValueError("LoadedModel.list_voxels: vox_origin without coordinates (xyz=False)")
        origin = None
        if vox_origin is not None:
            origin = np.ascontiguousarray(np.asarray(vox_origin, dtype=np.float64).reshape(-1))
            if origin.shape != (3,):
                raise ValueError("LoadedModel.list_voxels: vox_origin must hold 3 values")
        if out is not None and ((out.B, out.N, out.capacity) != (n, N, cap) or (out.xyz is not None) != bool(xyz)):
            raise ValueError("LoadedModel.list_voxels: `out` was made for another n, capacity or xyz")
        if out is None:
            # n < 1 (or no run yet) is the library's to refuse; the list it is refused with still has one item
            out = VoxelList(max(n, 1), N, cap, bool(xyz), torch.device("cuda", torch.cuda.current_device()))
        out._counts = None
        vo = _lib.VoxelOut(capacity=cap, voxel_size=0.0 if voxel_size is None else float(voxel_size),
                           origin=None if origin is None else origin.ctypes.data, count=out.count.data_ptr(),
                           hist=out.hist.data_ptr(), index=out.index.data_ptr(), cls=out.cls.data_ptr(),
                           xyz=_ptr(out.xyz))
        st = _stream_for(stream, [out.count, out.hist, out.index, out.cls, out.xyz])
        _lib.check(_lib.lib().occd_model_list_voxels(self.handle, n, C.byref(vo), st), "occd_model_list_voxels")
        return out

    def close(self):
        if self.handle:
            _lib.lib().occd_model_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


def run_frame_group(models, frame, out=None, stream=None, graph=True, conf=None):
    """one frame through every rank of a local group (LoadedModel r loaded with Comm.local(world)[r]), in lock step
    on one stream (occd_model_run_frame_group) -> rank 0's whole map, or (map, conf), as LoadedModel.run_frame"""
    hs = (C.c_void_p * len(models))(*[m.handle.value for m in models])
    f, keep, out, conf_t, st = _frame_call(models[0].geom, frame, out, stream, graph, conf, True, "rgb",
                                           "deploy.run_frame_group")
    for m in models:
        m._last_n = 0
    _lib.check(_lib.lib().occd_model_run_frame_group(hs, len(models), C.byref(f), _ptr(out), _ptr(conf_t), st),
               "occd_model_run_frame_group")
    for m in models:
        m._last_n = 1
    return out if conf is None else (out, conf_t)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _frame_call(g, frame, out, stream, graph, conf, root, pixel_format, who):
    """the occd_frame of a predict_frame frame dict whose images are in `pixel_format` (with the host and device
    copies it points into, which must live until the call returns; keep[0] is the images), the outputs (allocated when
    not given; none on a slab rank other than 0) and the stream.  The images must be the model's V views of that
    format: the library reads them from their shape."""
    if frame.get("pixel_format", pixel_format) != pixel_format:
        raise ValueError("%s: the frame's pixel_format is %r, this call stages %r"
                         % (who, frame["pixel_format"], pixel_format))
    if frame.get("rect_maps") is not None:
        raise ValueError("%s: a model file rectifies with the maps it was exported with; the frame's rect_maps would "
                         "be ignored" % who)
    img = torch.as_tensor(frame["img"])
    nv12 = pixel_format == "nv12"
    if img.dim() == (2 if nv12 else 3):
        img = img.unsqueeze(0)
    if (img.dtype != torch.uint8 or img.shape[0] != g.V
            or (img.dim() != 3 or img.shape[1] % 3 or img.shape[2] % 2 if nv12
                else img.dim() != 4 or img.shape[3] != 3)):
        raise ValueError("%s: frame['img'] must be the model's %d uint8 images, %s" % (
            who, g.V, "(V, H * 3 / 2, W) NV12 with H and W even" if nv12 else "(V, H, W, 3) %s" % pixel_format.upper()))
    img = img.contiguous().cuda()
    keep = [img]

    def host(a, dt=np.float64):
        a = np.ascontiguousarray(np.asarray(a, dt))
        keep.append(a)
        return a.ctypes.data

    f = _lib.Frame()
    # NV12: the luma plane's size; the chroma rows follow it (uv_offset = H0 rows)
    H0 = img.shape[1] * 2 // 3 if pixel_format == "nv12" else img.shape[1]
    f.images, f.H0, f.W0 = img.data_ptr(), H0, img.shape[2]
    f.img_stride, f.row_stride = img.stride(0), img.stride(1)
    # a float32 pose is applied in float32, as predict_frame does; cam_k then goes in the same type
    pose = np.asarray(frame["cam_pose"] if g.dataset == 1 else frame["T_velo_2_cam"])
    f.calib_f32 = 1 if pose.dtype == np.float32 else 0
    cdt = np.float32 if f.calib_f32 else np.float64
    if g.dataset == 1:
        f.pose = host(np.linalg.inv(pose), cdt)
        f.cam_k = host(frame["cam_k"], cdt) if "cam_k" in frame else None
        f.vox_origin = host(frame["vox_origin"])
        if g.has_depth:
            d = torch.as_tensor(frame["depth"]).contiguous().cuda()
            keep.append(d)
            f.depth, f.depth_h, f.depth_w = d.data_ptr(), d.shape[0], d.shape[1]
    else:
        f.cam_k, f.pose = host(frame["cam_k"], cdt), host(pose, cdt)
        if "vox_origin" in frame:
            f.vox_origin = host(frame["vox_origin"])
    if "scene_size" in frame:
        f.scene_size = host(frame["scene_size"])
    f.voxel_size = float(frame.get("voxel_size", 0.0))
    f.flags = 0 if graph else _lib.FRAME_NO_GRAPH
    if not root:
        out = conf = None
    else:
        if out is None:
            out = torch.empty(1, g.X, g.Y, g.Z, dtype=torch.uint16, device=img.device)
        if conf is True:
            conf = torch.empty(1, g.X, g.Y, g.Z, dtype=torch.float16, device=img.device)
        if conf is not None:
            assert conf.dtype == torch.float16 and conf.is_cuda and conf.is_contiguous() and conf.numel() == out.numel()
    return f, keep, out, conf, _stream_for(stream, [k for k in keep if isinstance(k, torch.Tensor)] + [out, conf])


def _stream_for(stream, tensors):
    """the launch stream of a run; on a stream of the caller's, the inputs copied and outputs allocated on the current
    stream must live until that stream is done"""
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
        for t in tensors:
            if t is not None:
                t.record_stream(stream)
    return C.c_void_p((stream or torch.cuda.current_stream()).cuda_stream)
