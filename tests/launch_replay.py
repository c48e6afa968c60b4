"""Per-launch parity of the non-convolution launches: one recorded library call of a planned model, replayed alone, in
place, against float64.  The sibling of tests/conv_replay.py, shared by tests/test_launch_replay_host.py and
tests/test_gpu_launch_replay.py (a plain helper, imported like gpu_cases).

  Recording(m)        installs deploy._Recorder BEFORE the plan is built (a plan's FnOps capture `_lib.lib()` when
                      they are built), so running the plan's non-ConvOp ops with `recording = True` afterwards yields
                      every non-convolution call it makes as (entry point, typed arguments).  occd_conv_run (the conv
                      replay covers it) and occd_comm_* (the slab tests cover them) are dropped.
  Storages(tensors)   every device storage a plan holds; a recorded pointer becomes (storage, byte offset)
  signature(rec, st)  entry point, every scalar argument, and for each pointer its storage size and byte offset (an
                      sfa_params blob: every field, pointers likewise): equal signatures are the same launch on
                      different data
  SPECS[name]         per entry point, written from include/occdepth_b200.h: the regions it reads (channel windows of
                      [positions][cstride] buffers, planar tensors, tables), the regions it writes (output windows
                      over roundup(C, 8) channels where the kernel stores 8-channel vectors; the squeeze `pool` it
                      accumulates into; the per-image weight sets and `hidden` of the SE fold, and `pool`, which the fold
                      zeroes; in-place operands: occd_channel_scale's x, the tapsum's out when pre == out), and the
                      float64 reference of every output
  check(...)          conv_replay's element-wise form  |got - ref| <= 1/2 ulp_store(|ref| + d) + d,  d = C sqrt(K) S
                      (+ A |v| for SiLU): K the terms of one output's sum, S the sum of their absolute values, stores
                      rounded the storage type's way (TF32 to nearest, ties away; bf16 to nearest even; fp32 where the
                      header says fp32).  Per entry point:
                        copy_channels, cl_transpose   bit-exact
                        dwconv (depthwise)            K = k*k taps + bias; SiLU with conv_replay's slope and A_ACT
                        squeeze (its pool)            pool_after - pool_before against 2^24 sum of the device's STORED
                                                      outputs: 1/2 per contributing block (its __float2ll_rn) plus the
                                                      fp32 partial-sum term
                        SE fold                       hidden (K = C + 1, SiLU) in fp32; wout = round_wdtype(master *
                                                      gate) with the gate's error carried by |master| (1 + sqrt(R) S2);
                                                      pool zero afterwards; pad columns [C, Kpad) zero
                        bilinear / tapsum             K = 4 / 9 taps x 4 corners (+ pre); S also holds each corner
                                                      pair's difference times its fp32 source coordinate (the kernels
                                                      compute the coordinates in fp32, as PyTorch's kernel does)
                        virtual view                  K = 4 corners of grid_sample(border); S as for the resize, the
                                                      coordinate being the disparity-shifted fp32 one
                        lift, prior (both routes)     the restatements' own bound: C max|ref| of the launch
                        softmax(_to_cl), fc           K = C (S = the probability) / K = n_in + 1
                        channel_scale                 one fp32 product, one rounding
  NOTHING ELSE MOVES: every byte of every storage the launch reaches equals its state before the launch, except the
  declared output regions.

Pointers arrive as they are recorded, so a window's channel offset lives in its pointer: a [positions][cstride] input
read at pointer p over C channels is rows [p + r cstride, p + r cstride + C), and the channels the launch must NOT read
are [p + r cstride + C, p + (r + 1) cstride) -- channels [coff + C, cstride) of row r and [0, coff) of row r + 1.

The constants are at most twice the largest ratio seen over the sweep of tests/test_gpu_launch_replay.py on an
NVIDIA H100 80GB HBM3 (power limit 700 W); see C_ACC below.  The prior's (2.02e-5 of max|ref| at KITTI's 1370 x 376
frustum) is above the 1.6e-5 that tests/test_gpu_ops_edges.py measured at its synthetic 320 x 96 one: the fp32 frustum
coordinates lose more at the real image size.
"""
import bisect
import contextlib
import ctypes as C
import types

import torch
import torch.nn.functional as F

import conv_replay as CR
from conv_replay import quantize, ulp_store  # noqa: F401  (re-exported: the stores of every entry point)

f64 = torch.float64
SKIP_PREFIX = ("occd_conv_run", "occd_comm_")

# per comparator family and precision: the constant in front of sqrt(K) S (module docstring).  Each is at most twice
# the largest (|got - ref| - 1/2 ulp) / (sqrt(K) S) seen over the sweep of tests/test_gpu_launch_replay.py (all six
# shipped configurations, both precisions, forward + class-map + two slab rank plans + infer_mode + two NYU frames:
# 480 distinct launches) on an NVIDIA H100 80GB HBM3 (power limit 700 W), which found no failing launch:
#   tf32: fc 1.51e-8, lift 1.57e-7, pool 5.4e-9, prior 2.02e-5, resize 6.71e-8, se 5.51e-8, softmax 7.81e-8,
#         vview 6.12e-8
#   bf16: lift 1.75e-7, pool 1.93e-9, resize 5.42e-8, se 3.62e-8, softmax 4.43e-8, vview 5.81e-8, SiLU (tanh.approx)
#         3.02e-6 per |v|
# Launches whose arguments do not depend on the precision (the fp32 DepthNet helpers and the prior) are replayed once,
# in the tf32 sweep: their bf16 constants are the tf32 ones.  The depthwise launches all end in SiLU, whose ratio
# nets out the accumulation term (conv_replay's form): for tf32 it stayed below zero, so "dw" keeps conv_replay's
# accumulation constant and the SiLU gets no term of its own; likewise the SE MLP's SiLU (ratio -6.0e-7).
C_ACC = {
    "dw": {"tf32": 6.0e-8, "bf16": 6.0e-8},
    "pool": {"tf32": 1.0e-8, "bf16": 3.8e-9},
    "se": {"tf32": 1.1e-7, "bf16": 7.0e-8},
    "resize": {"tf32": 1.3e-7, "bf16": 1.0e-7},
    "vview": {"tf32": 1.2e-7, "bf16": 1.1e-7},
    "softmax": {"tf32": 1.5e-7, "bf16": 8.8e-8},
    "fc": {"tf32": 3.0e-8, "bf16": 3.0e-8},
    "lift": {"tf32": 3.1e-7, "bf16": 3.5e-7},
    "prior": {"tf32": 4.0e-5, "bf16": 4.0e-5},
}
A_ACT = {"tf32": dict(), "bf16": dict(silu=6.0e-6)}      # the bf16 depthwise SiLU (tanh.approx)
A_SE = 0.0                                                # the SE MLP's SiLU: covered by the accumulation term

STORE = {0: "tf32", 1: "bf16"}
TDT = {0: torch.float32, 1: torch.bfloat16}
ACT = {0: "none", 1: "relu", 2: "leaky", 3: "silu", 4: "sigmoid"}


def _r8(c):
    return (c + 7) // 8 * 8


# ---------------------------------------------------------------------------------------------------------------
# recording
class Recording:
    """context manager: deploy._Recorder stands in for the library on this thread while it is open.  Build (and run)
    the plan inside it, then calls(plan) records the plan's non-convolution launches without running them."""

    def __enter__(self):
        from occdepth_b200 import _lib, deploy
        self.rec = deploy._Recorder(_lib.lib())
        _lib._RECORDING.recorder = self.rec
        return self

    def __exit__(self, *exc):
        from occdepth_b200 import _lib
        _lib._RECORDING.recorder = None

    def calls(self, plan):
        from occdepth_b200 import deploy
        from occdepth_b200.engine import ConvOp
        self.rec.calls = []
        self.rec.recording = True
        try:
            for op in plan.ops:
                if not isinstance(op, ConvOp):
                    op.run(deploy._STREAM)
        finally:
            self.rec.recording = False
        return [(n, a) for n, a in self.rec.calls if not n.startswith(SKIP_PREFIX)]


def plan_tensors(plan, extra=()):
    """every tensor a plan holds: its ops' kept tensors, its convolutions' operands, its FlospDepth state"""
    from occdepth_b200 import deploy
    from occdepth_b200.engine import ConvOp
    out = []
    for op in plan.ops:
        deploy._collect(getattr(op, "_keep", ()), out)
        if isinstance(op, ConvOp):
            out += [t for _, t in CR.reach(op)]
    deploy._collect([getattr(plan, "flosp_state", None), list(extra)], out)
    return out


class Storages:
    """the storages behind a plan's tensors; place(p) -> (storage key, byte offset)"""

    def __init__(self, tensors):
        self.by_key = {}
        for t in tensors:
            s = t.untyped_storage()
            if s.nbytes():
                self.by_key.setdefault(s.data_ptr(), s)
        self.keys = sorted(self.by_key)

    def place(self, p, what=""):
        k = bisect.bisect_right(self.keys, p) - 1
        if k < 0 or not p < self.keys[k] + self.by_key[self.keys[k]].nbytes():
            raise KeyError("%s: pointer 0x%x lands in no storage the plan holds" % (what, p))
        return self.keys[k], p - self.keys[k]

    def nbytes(self, key):
        return self.by_key[key].nbytes()


def sfa_params(blob):
    """an ("h", blob) argument of occd_sfa_lift_fwd back into occd_sfa_params, its pointers restored"""
    from occdepth_b200 import _lib
    data, ptrs = blob
    p = _lib.SfaParams.from_buffer_copy(data)
    for off, v in ptrs:
        C.c_uint64.from_address(C.addressof(p) + off).value = v
    return p


def _pointer_fields(p):
    return ([("feat%d" % i, p.feat[i]) for i in range(p.n_scales)] + [("pix", p.pix), ("fov", p.fov), ("out", p.out),
                                                                      ("prior", p.prior)])


def named(rec):
    """(entry point, typed args) -> dict of argument name -> value (pointers as ints, 0 for NULL)"""
    name, args = rec
    names = SPECS[name].args
    assert len(names) == len(args), (name, len(args))
    out = {}
    for n, a in zip(names, args):
        if a[0] in ("i", "l", "f", "d", "p"):
            out[n] = a[1]
        elif a[0] == "n":
            out[n] = 0
        elif a[0] == "h":
            out[n] = sfa_params(a[1])
    return out


def signature(rec, st):
    name, args = rec
    sig = [name]
    for a in args:
        if a[0] == "p":
            k, off = st.place(a[1], name)
            sig.append(("p", st.nbytes(k), off))
        elif a[0] == "h":
            p = sfa_params(a[1])
            fields = []
            for f, _ in p._fields_:
                v = getattr(p, f)
                fields.append((f, tuple(v) if isinstance(v, C.Array) else v))
            ptrs = tuple((f, None if not v else (st.nbytes(st.place(v)[0]), st.place(v)[1]))
                         for f, v in _pointer_fields(p))
            sig.append(("h", tuple((f, v) for f, v in fields if f not in ("feat", "pix", "fov", "out", "prior")),
                        ptrs))
        elif a[0] == "s":
            sig.append(("s",))
        else:
            sig.append(tuple(a))
    return tuple(sig)


def call(rec, stream):
    """run the recorded launch through the real library on `stream` -> return code"""
    from occdepth_b200 import _lib
    name, args = rec
    vals = []
    for a in args:
        if a[0] in ("i", "l", "f", "d", "p"):
            vals.append(a[1])
        elif a[0] == "n":
            vals.append(None)
        elif a[0] == "s":
            vals.append(stream)
        elif a[0] == "h":
            vals.append(C.byref(sfa_params(a[1])))
        else:
            raise ValueError("cannot replay argument %r of %s" % (a, name))
    return getattr(_lib.lib(), name)(*vals)


# ---------------------------------------------------------------------------------------------------------------
# regions of storages
class Reg:
    """elements of one storage: byte offset, element shape and strides, dtype.  win: for a channels-last input, the
    count C of channels read at the start of each row of `cstride` elements (rows are dim -2 ... of the view)"""

    def __init__(self, key, off, shape, stride, dtype, win=None, inplace=False):
        self.key, self.off, self.shape, self.stride, self.dtype = key, off, tuple(shape), tuple(stride), dtype
        self.win, self.inplace = win, inplace

    def view(self, storages):
        s = storages[self.key]
        es = torch.empty(0, dtype=self.dtype).element_size()
        assert self.off % es == 0, (self.off, es)
        return torch.empty(0, dtype=self.dtype, device=s.device).set_(s, self.off // es, self.shape, self.stride)

    def byte_mask(self, mask):
        """mark the region's bytes in the uint8 mask of its storage"""
        es = torch.empty(0, dtype=self.dtype).element_size()
        v = mask.as_strided(self.shape + (es,), tuple(x * es for x in self.stride) + (1,), self.off)
        v.fill_(1)


def cl(st, p, rows, cstride, C_, dtype, inplace=False):
    """rows x [cstride] channels-last rows starting at pointer p, C_ channels read / written at the start of each"""
    k, off = st.place(p)
    return Reg(k, off, (rows, C_), (cstride, 1), dtype, win=(C_, cstride), inplace=inplace)


def flat(st, p, n, dtype, inplace=False):
    k, off = st.place(p)
    return Reg(k, off, (n,), (1,), dtype, inplace=inplace)


# ---------------------------------------------------------------------------------------------------------------
# references (float64), written from include/occdepth_b200.h
def activation(v, act):
    return CR.activation(v, act)


def dwconv_ref(x, w, bias, K, S, pad_top, pad_left, OH, OW, act):
    """x float64 [B, H, W, C]; w [K*K, C]; -> (out, v, Ssum) [B, OH, OW, C]: TF-SAME depthwise conv with explicit
    top / left padding (zero outside the map), bias, activation"""
    B, H, W, C_ = x.shape
    v = bias.expand(B, OH, OW, C_).clone()
    Sm = bias.abs().expand(B, OH, OW, C_).clone()
    for ky in range(K):
        for kx in range(K):
            iy = torch.arange(OH, device=x.device) * S - pad_top + ky
            ix = torch.arange(OW, device=x.device) * S - pad_left + kx
            my, mx = (iy >= 0) & (iy < H), (ix >= 0) & (ix < W)
            g = x[:, iy.clamp(0, H - 1)][:, :, ix.clamp(0, W - 1)] * (my[:, None] & mx[None, :])[None, :, :, None]
            t = g * w[ky * K + kx]
            v += t
            Sm += t.abs()
    return activation(v, act), v, Sm


def _bilinear_ac_axis(n_out, n_in, dev):
    """align_corners=True source coordinate per output index (float64), its lower / upper index and weight"""
    s = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    f = torch.arange(n_out, device=dev, dtype=f64) * s
    i0 = f.floor().long().clamp(max=n_in - 1)
    i1 = (i0 + 1).clamp(max=n_in - 1)
    return f, i0, i1, f - i0


def bilinear_ac_ref(x, OH, OW):
    """F.interpolate(bilinear, align_corners=True) of float64 [B, h, w, C] -> (out, S) [B, OH, OW, C]; S: the sum of
    the corner terms' absolute values plus each corner pair's difference times its source coordinate (the scale of
    an fp32 coordinate's error)"""
    B, h, w, C_ = x.shape
    fy, y0, y1, ly = _bilinear_ac_axis(OH, h, x.device)
    fx, x0, x1, lx = _bilinear_ac_axis(OW, w, x.device)
    ly, lx = ly[None, :, None, None], lx[None, None, :, None]
    r0, r1 = x[:, y0], x[:, y1]
    a, b, c, d = r0[:, :, x0], r0[:, :, x1], r1[:, :, x0], r1[:, :, x1]
    top = (1 - lx) * a + lx * b
    bot = (1 - lx) * c + lx * d
    out = (1 - ly) * top + ly * bot
    S = ((1 - ly) * ((1 - lx) * a.abs() + lx * b.abs()) + ly * ((1 - lx) * c.abs() + lx * d.abs())
         + fy[None, :, None, None] * (bot - top).abs()
         + fx[None, None, :, None] * ((1 - ly) * (b - a).abs() + ly * (d - c).abs()))
    return out, S


def tapsum_ref(ys, pre, OH, OW, act):
    """ys: nine float64 [B, h, w, C] (tap t = (dy+1)*3 + (dx+1)), pre float64 [B, OH, OW, C] or None ->
    (out, v, S): out[p] = act(pre[p] + sum_t [p+t inside] bilinear_ac(Y_t)(p+t))"""
    v = torch.zeros(ys[0].shape[0], OH, OW, ys[0].shape[-1], dtype=f64, device=ys[0].device)
    Sm = torch.zeros_like(v)
    if pre is not None:
        v += pre
        Sm += pre.abs()
    for t, y in enumerate(ys):
        dy, dx = t // 3 - 1, t % 3 - 1
        r, s = bilinear_ac_ref(y, OH, OW)
        ya, yb = max(0, -dy), min(OH, OH - dy)          # output rows whose p + t is inside
        xa, xb = max(0, -dx), min(OW, OW - dx)
        v[:, ya:yb, xa:xb] += r[:, ya + dy:yb + dy, xa + dx:xb + dx]
        Sm[:, ya:yb, xa:xb] += s[:, ya + dy:yb + dy, xa + dx:xb + dx]
    return activation(v, act), v, Sm


def softmax_ref(x, dim):
    m = x.max(dim, keepdim=True).values
    e = (x - m).exp()
    return e / e.sum(dim, keepdim=True)


def se_mlp_ref(pool, inv_hw, w1, b1, w2t, b2):
    """pool int64 [B, C] (2^-24 units) -> (hidden, gate, S1, S2) float64: hidden = silu(W1 mean + b1), gate =
    sigmoid(W2 hidden + b2), mean = pool 2^-24 inv_hw; S1 / S2 the sums of absolute terms"""
    mean = pool.to(f64) * 2.0 ** -24 * float(inv_hw)
    a1 = mean @ w1.t() + b1
    S1 = mean.abs() @ w1.abs().t() + b1.abs()
    hidden = a1 * torch.sigmoid(a1)
    a2 = hidden @ w2t + b2
    S2 = hidden.abs() @ w2t.abs() + b2.abs()
    return hidden, torch.sigmoid(a2), a1, S1, S2


def lift_ref(feats, divs, pix, fov, perm=None, prior=None, scale_const=1.0):
    """feats: per scale float64 [V, h, w, C]; pix [V, N, P, 2] int64; fov [V, N, P] bool -> float64 [N, C] in output
    voxel order.  Per scale and view: mean over the in-FOV points of feat[(y // div) * w + (x // div)] (floor
    division; an index outside the map contributes zero but its point still counts), mask = any point in FOV; views
    are combined by the pairwise cosine soft-assignment of SFA.forward; scales are summed."""
    V, N, P, _ = pix.shape
    Cc = feats[0].shape[3]
    dev = feats[0].device
    pix, fov = pix.to(dev), fov.to(dev)
    out = torch.zeros(N, Cc, dtype=torch.float64, device=dev)
    for f, d in zip(feats, divs):
        h, w = f.shape[1], f.shape[2]
        idx = torch.div(pix[..., 1], d, rounding_mode="floor") * w + torch.div(pix[..., 0], d, rounding_mode="floor")
        inmap = (idx >= 0) & (idx < h * w)
        fs, ms = [], []
        for v in range(V):
            g = f[v].reshape(h * w, Cc)[idx[v].clamp(0, h * w - 1)]                # [N, P, C]
            g = g * (fov[v] & inmap[v]).unsqueeze(-1).double()
            cnt = fov[v].sum(1)
            fs.append(g.sum(1) / cnt.clamp_min(1).unsqueeze(-1).double())
            ms.append((cnt > 0).double())
        if V == 1:
            out += fs[0]
            continue
        acc = torch.zeros_like(out)
        for a in range(V):
            for b in range(a + 1, V):
                cos = (fs[a] * fs[b]).sum(1) / (fs[a].norm(dim=1).clamp_min(1e-8) * fs[b].norm(dim=1).clamp_min(1e-8))
                cos = cos * ms[a] * ms[b]
                wa = cos + (ms[a] > ms[b]).double()
                wb = cos + (ms[b] > ms[a]).double()
                acc += wa.unsqueeze(1) * fs[a] + wb.unsqueeze(1) * fs[b]
        out += acc / (V * (V - 1))
    n = torch.arange(N, device=dev)
    no = n
    if perm is not None:
        S1, S2 = perm
        no = (n // (S1 * S2) * S1 + n % S1) * S2 + (n // S1) % S2
    res = torch.empty_like(out)
    res[no] = out
    if prior is not None:
        res = res * prior.double().unsqueeze(1) * scale_const
    return res


def frustum_grid_f64(TG, K4, ida, grid, img_hw, Dn, dmin, dmax, x0=0, Xl=None):
    """oracle.functional.frustum_grid restated in float64 over X planes [x0, x0 + Xl) of `grid` (X, Y, Z): TG = the
    4x4 lidar->camera transform times grid->lidar, K4 the 4x4 intrinsics (rows 0..2 used), ida 4x4 ->
    normalised sampling coordinates [1, Xl, Y, Z, 3]"""
    X, Y, Z = grid
    Xl = X - x0 if Xl is None else Xl
    d = torch.float64
    TG, K4, ida = TG.double(), K4.double(), ida.double()
    dev = TG.device
    i, j, k = torch.meshgrid(torch.arange(x0, x0 + Xl, dtype=d, device=dev), torch.arange(Y, dtype=d, device=dev),
                             torch.arange(Z, dtype=d, device=dev), indexing="ij")
    vox = torch.stack([i, j, k, torch.ones_like(i)], -1)
    vox[..., :3] += 0.5

    def dehom(p):
        z = p[..., -1:]
        return p[..., :-1] * torch.where(z.abs() > 1e-8, 1.0 / (z + 1e-8), torch.ones_like(z))

    cam = dehom(vox @ TG.t())
    pt = F.pad(cam, [0, 1], value=1.0) @ K4[:3].t()
    img = dehom(pt)
    depth = pt[..., 2] - K4[2, 3]
    bin_size = 2 * (dmax - dmin) / (Dn * (1 + Dn))
    idx = -0.5 + 0.5 * torch.sqrt(1 + 8 * (depth - dmin) / bin_size)
    fg = dehom(F.pad(torch.cat([img, idx.unsqueeze(-1)], -1), [0, 1], value=1.0) @ ida.t())
    fg = fg / (torch.tensor([img_hw[1], img_hw[0], Dn], dtype=d, device=dev) - 1) * 2 - 1
    fg[~torch.isfinite(fg)] = -2
    return fg.unsqueeze(0)


def sample_mean(depth, grids, mean_mode):
    """F.grid_sample of each view's depth volume and of an all-ones volume, then the masked mean"""
    V = depth.shape[0]
    fs = [F.grid_sample(depth[v][None, None], grids[v], mode="bilinear", padding_mode="zeros", align_corners=False)
          for v in range(V)]
    ms = [F.grid_sample(torch.ones_like(depth[v])[None, None], grids[v], mode="bilinear", padding_mode="zeros",
                        align_corners=False) for v in range(V)]
    agg, m = sum(fs), sum(ms)
    if V > 1 and mean_mode:
        agg = torch.where(m > 0, agg / m, agg)
    return agg.reshape(-1), m.reshape(-1)


def virtual_view_ref(x, depth, bf_scale):
    """OccDepth.generate_virtual_img (the reference's OccDepth.py:233-260) in float64 for one item: x [h, w, C],
    depth [dh, dw] -> (out, S) [h, w, C].  Depth resized bilinearly (align_corners=False) to h x w, disparity
    bf_scale / depth (inf -> 0), base grid -1 + 2x/w shifted by disparity * 2 / w, grid_sample(bilinear, border,
    align_corners=False).  S: corner terms plus each corner pair's difference times the coordinate's magnitude."""
    h, w, _ = x.shape
    dh, dw = depth.shape
    d = F.interpolate(depth[None, None].double(), size=(h, w), mode="bilinear", align_corners=False)[0, 0]
    dx = bf_scale / d
    dx = torch.where(torch.isinf(dx), torch.zeros_like(dx), dx)
    xs = torch.arange(w, dtype=f64, device=x.device)
    ys = torch.arange(h, dtype=f64, device=x.device)
    gx = -1 + 2 * xs[None, :] / w + dx * 2 / w
    gy = (-1 + 2 * ys / h)[:, None].expand(h, w)
    fx = (((gx + 1) * w - 1) / 2).clamp(0, w - 1)
    fy = (((gy + 1) * h - 1) / 2).clamp(0, h - 1)
    ix0, iy0 = fx.floor().long(), fy.floor().long()
    ix1, iy1 = (ix0 + 1).clamp(max=w - 1), (iy0 + 1).clamp(max=h - 1)
    tx, ty = (fx - ix0)[..., None], (fy - iy0)[..., None]
    a, b, c, e = x[iy0, ix0], x[iy0, ix1], x[iy1, ix0], x[iy1, ix1]
    top, bot = (1 - tx) * a + tx * b, (1 - tx) * c + tx * e
    out = (1 - ty) * top + ty * bot
    S = ((1 - ty) * ((1 - tx) * a.abs() + tx * b.abs()) + ty * ((1 - tx) * c.abs() + tx * e.abs())
         + (w + dx.abs())[..., None] * ((1 - ty) * (b - a).abs() + ty * (e - c).abs())
         + float(h) * (bot - top).abs())
    return out, S


# ---------------------------------------------------------------------------------------------------------------
# per entry point: argument names, the regions read and written, the float64 outputs
class Out(types.SimpleNamespace):
    """one output to compare: reg, ref (float64, the region's shape), S, K, family, store, act, v; exact: bits"""


def _vec_dtype(a):
    return TDT[a["dtype"]]


def _spec_dwconv(a, st):
    dt = _vec_dtype(a)
    B, H, W, OH, OW, C_ = a["B"], a["H"], a["W"], a["OH"], a["OW"], a["C"]
    Cw = _r8(C_)
    reads = [cl(st, a["in"], B * H * W, a["cs_in"], Cw, dt), flat(st, a["w"], a["K"] ** 2 * C_, torch.float32),
             flat(st, a["bias"], C_, torch.float32)]
    writes = [cl(st, a["out"], B * OH * OW, a["cs_out"], Cw, dt)]
    if a["pool"]:
        writes.append(Reg(*st.place(a["pool"]), (B, C_), (C_, 1), torch.int64, inplace=True))
    return reads, writes


def _ref_dwconv(a, R, W, prec):
    B, H, Wd, OH, OW, C_ = a["B"], a["H"], a["W"], a["OH"], a["OW"], a["C"]
    x = R[0][:, :C_].to(f64).view(B, H, Wd, C_)
    out, v, S = dwconv_ref(x, R[1].to(f64).view(-1, C_), R[2].to(f64), a["K"], a["stride"], a["pad_top"],
                           a["pad_left"], OH, OW, ACT[a["act"]])
    sh = (B * OH * OW, C_)
    outs = [Out(idx=0, cols=C_, ref=out.reshape(sh), S=S.reshape(sh), K=a["K"] ** 2 + 1, family="dw",
                store=STORE[a["dtype"]], act=ACT[a["act"]], v=v.reshape(sh))]
    if a["pool"]:
        outs.append(Out(idx=1, pool=True, OH=OH, OW=OW, B=B, C=C_))
    return outs


def _spec_se_fold(a, st):
    B, C_, R_, rows, Kpad = a["B"], a["C"], a["R"], a["rows"], a["Kpad"]
    reads = [Reg(*st.place(a["pool"]), (B, C_), (C_, 1), torch.int64, inplace=True),
             flat(st, a["w1"], R_ * C_, torch.float32), flat(st, a["b1"], R_, torch.float32),
             flat(st, a["w2t"], R_ * C_, torch.float32), flat(st, a["b2"], C_, torch.float32),
             flat(st, a["master"], rows * Kpad, torch.float32)]
    writes = [Reg(*st.place(a["pool"]), (B, C_), (C_, 1), torch.int64, inplace=True),
              flat(st, a["hidden"], B * R_, torch.float32),
              flat(st, a["wout"], B * rows * Kpad, TDT[a["wdtype"]])]
    return reads, writes


def _ref_se_fold(a, R, W, prec):
    B, C_, R_, rows, Kpad = a["B"], a["C"], a["R"], a["rows"], a["Kpad"]
    hidden, gate, a1, S1, S2 = se_mlp_ref(R[0], a["inv_hw"], R[1].to(f64).view(R_, C_), R[2].to(f64),
                                          R[3].to(f64).view(R_, C_), R[4].to(f64))
    master = R[5].to(f64).view(rows, Kpad)
    ref = torch.zeros(B, rows, Kpad, dtype=f64, device=master.device)
    ref[:, :, :C_] = master[None, :, :C_] * gate[:, None, :]
    S = torch.zeros_like(ref)
    S[:, :, :C_] = master[None, :, :C_].abs() * (1 + R_ ** 0.5 * S2[:, None, :])
    return [Out(idx=0, zero=True),
            Out(idx=1, ref=hidden.reshape(-1), S=S1.reshape(-1), K=C_ + 1, family="se", store="fp32", act="silu",
                v=a1.reshape(-1), a_act=A_SE),
            Out(idx=2, ref=ref.reshape(-1), S=S.reshape(-1), K=1, family="se", store=STORE[a["wdtype"]],
                act="none")]


def _spec_bilinear(a, st):
    dt = _vec_dtype(a)
    B, h, w, OH, OW, Cw = a["B"], a["h"], a["w"], a["OH"], a["OW"], _r8(a["C"])
    es = torch.empty(0, dtype=dt).element_size()
    reads = [cl(st, a["in"] + a["in_off"] * es, B * h * w, a["cs_in"], Cw, dt)]
    writes = [cl(st, a["out"] + a["out_off"] * es, B * OH * OW, a["cs_out"], Cw, dt)]
    return reads, writes


def _ref_bilinear(a, R, W, prec):
    B, h, w, OH, OW, Cw = a["B"], a["h"], a["w"], a["OH"], a["OW"], _r8(a["C"])
    out, S = bilinear_ac_ref(R[0].to(f64).view(B, h, w, Cw), OH, OW)
    sh = (B * OH * OW, Cw)
    return [Out(idx=0, ref=out.reshape(sh), S=S.reshape(sh), K=4, family="resize", store=STORE[a["dtype"]],
                act="none")]


def _spec_tapsum(a, st):
    dt = _vec_dtype(a)
    B, h, w, OH, OW, Cw = a["B"], a["h"], a["w"], a["OH"], a["OW"], _r8(a["C"])
    es = torch.empty(0, dtype=dt).element_size()
    reads = [cl(st, a["y"] + (a["y_off"] + t * a["tap_stride"]) * es, B * h * w, a["cs_y"], Cw, dt)
             for t in range(9)]
    inplace = bool(a["pre"]) and a["pre"] + a["pre_off"] * es == a["out"] + a["out_off"] * es
    if a["pre"]:
        reads.append(cl(st, a["pre"] + a["pre_off"] * es, B * OH * OW, a["cs_pre"], Cw, dt, inplace=inplace))
    writes = [cl(st, a["out"] + a["out_off"] * es, B * OH * OW, a["cs_out"], Cw, dt, inplace=inplace)]
    return reads, writes


def _ref_tapsum(a, R, W, prec):
    B, h, w, OH, OW, Cw = a["B"], a["h"], a["w"], a["OH"], a["OW"], _r8(a["C"])
    ys = [R[t].to(f64).view(B, h, w, Cw) for t in range(9)]
    pre = R[9].to(f64).view(B, OH, OW, Cw) if a["pre"] else None
    out, v, S = tapsum_ref(ys, pre, OH, OW, ACT[a["act"]])
    sh = (B * OH * OW, Cw)
    return [Out(idx=0, ref=out.reshape(sh), S=S.reshape(sh), K=37, family="resize", store=STORE[a["dtype"]],
                act=ACT[a["act"]], v=v.reshape(sh))]


_LIFT_MODES = {0: ("fp32", torch.float32), 1: ("bf16", torch.bfloat16), 2: ("fp32", torch.float32),
               3: ("tf32", torch.float32)}


def _spec_lift(a, st):
    p = a["p"]
    V, Cc, N, P = p.n_views, p.C, p.N, p.P
    fdt = TDT[p.feat_dtype]
    reads = []
    for s in range(p.n_scales):
        vs = p.vstride[s] or p.h[s] * p.w[s] * Cc
        k, off = st.place(p.feat[s])
        reads.append(Reg(k, off, (V, p.h[s] * p.w[s], Cc), (vs, Cc, 1), fdt))
    reads += [flat(st, p.pix, V * N * P * 2, torch.int64), flat(st, p.fov, V * N * P, torch.uint8)]
    if p.prior:
        reads.append(flat(st, p.prior, N, torch.float32))
    _, odt = _LIFT_MODES[p.out_mode]
    if p.out_mode == 0:
        writes = [Reg(*st.place(p.out), (Cc, N), (N, 1), odt)]
    else:
        writes = [cl(st, p.out, N, p.out_cstride, Cc, odt)]
    return reads, writes


def _ref_lift(a, R, W, prec):
    p = a["p"]
    V, Cc, N, P = p.n_views, p.C, p.N, p.P
    feats = [R[s].to(f64).view(V, p.h[s], p.w[s], Cc) for s in range(p.n_scales)]
    ns = p.n_scales
    pix = R[ns].view(V, N, P, 2)
    fov = R[ns + 1].view(V, N, P).bool()
    prior = R[ns + 2] if p.prior else None
    ref = lift_ref(feats, [p.div[s] for s in range(ns)], pix, fov, perm=(p.S1, p.S2) if p.perm_nyu else None,
                   prior=prior, scale_const=p.scale_const if p.prior else 1.0)
    if p.out_mode == 0:
        ref = ref.t()
    S = torch.full_like(ref, float(ref.abs().max()) if ref.numel() else 0.0)
    return [Out(idx=0, ref=ref, S=S, K=1, family="lift", store=_LIFT_MODES[p.out_mode][0], act="none")]


def _cams_of(t):
    """one camera's 40 floats {T[12], K[12], ida[16]} -> (T 4x4 with a last row 0 0 0 1, K4, ida) float64"""
    t = t.to(f64)
    T = torch.eye(4, dtype=f64, device=t.device)
    T[:3] = t[:12].view(3, 4)
    K4 = torch.eye(4, dtype=f64, device=t.device)
    K4[:3] = t[12:24].view(3, 4)
    return T, K4, t[24:40].view(4, 4)


def _spec_prior(a, st):
    V, Dn, h, w, Y, Z, Xl = a["V"], a["Dn"], a["h"], a["w"], a["Y"], a["Z"], a["Xl"]
    reads = [flat(st, a["depth"], V * Dn * h * w, torch.float32)]
    if "cams" in a:
        reads.append(flat(st, a["cams"], V * 40, torch.float32))
    else:
        k, off = st.place(a["grids"])
        N = a["X"] * Y * Z
        reads.append(Reg(k, off + a["x0"] * Y * Z * 12, (V, Xl * Y * Z, 3), (N * 3, 3, 1), torch.float32))
    writes = [flat(st, a["out"], Xl * Y * Z, torch.float32)]
    return reads, writes


def _ref_prior(a, R, W, prec):
    V, Dn, h, w, X, Y, Z, x0, Xl = a["V"], a["Dn"], a["h"], a["w"], a["X"], a["Y"], a["Z"], a["x0"], a["Xl"]
    depth = R[0].to(f64).view(V, Dn, h, w)
    if "cams" in a:
        grids = []
        for v in range(V):
            T, K4, ida = _cams_of(R[1][v * 40:(v + 1) * 40])
            grids.append(frustum_grid_f64(T, K4, ida, (X, Y, Z), (a["img_h"], a["img_w"]), Dn, a["dmin"], a["dmax"],
                                          x0, Xl))
    else:
        grids = [R[1][v].to(f64).view(1, Xl, Y, Z, 3) for v in range(V)]
    ref, _ = sample_mean(depth, grids, a["mean_mode"])
    if a["perm_xzy"]:
        ref = ref.view(Xl, Y, Z).permute(0, 2, 1).reshape(-1)
    S = torch.full_like(ref, float(ref.abs().max()))
    return [Out(idx=0, ref=ref, S=S, K=1, family="prior", store="fp32", act="none")]


def _spec_softmax(a, st):
    B, C_, S_ = a["B"], a["C"], a["S"]
    return [flat(st, a["in"], B * C_ * S_, torch.float32)], [flat(st, a["out"], B * C_ * S_, torch.float32)]


def _ref_softmax(a, R, W, prec):
    B, C_, S_ = a["B"], a["C"], a["S"]
    p = softmax_ref(R[0].to(f64).view(B, C_, S_), 1).reshape(-1)
    return [Out(idx=0, ref=p, S=p, K=C_, family="softmax", store="fp32", act="none")]


def _spec_softmax_cl(a, st):
    B, C_, S_ = a["B"], a["C"], a["S"]
    dt = _vec_dtype(a)
    es = torch.empty(0, dtype=dt).element_size()
    return ([flat(st, a["in"], B * C_ * S_, torch.float32)],
            [cl(st, a["out"] + a["coff"] * es, B * S_, a["cstride"], C_, dt)])


def _ref_softmax_cl(a, R, W, prec):
    B, C_, S_ = a["B"], a["C"], a["S"]
    p = softmax_ref(R[0].to(f64).view(B, C_, S_), 1).permute(0, 2, 1).reshape(B * S_, C_)
    return [Out(idx=0, ref=p, S=p, K=C_, family="softmax", store=STORE[a["dtype"]], act="none")]


def _spec_fc(a, st):
    B, n_in, n_out = a["B"], a["n_in"], a["n_out"]
    return ([flat(st, a["in"], B * n_in, torch.float32), flat(st, a["w"], n_out * n_in, torch.float32),
             flat(st, a["bias"], n_out, torch.float32)], [flat(st, a["out"], B * n_out, torch.float32)])


def _ref_fc(a, R, W, prec):
    B, n_in, n_out = a["B"], a["n_in"], a["n_out"]
    x, w, b = R[0].to(f64).view(B, n_in), R[1].to(f64).view(n_out, n_in), R[2].to(f64)
    v = x @ w.t() + b
    S = x.abs() @ w.abs().t() + b.abs()
    act = ACT[a["act"]]
    return [Out(idx=0, ref=activation(v, act).reshape(-1), S=S.reshape(-1), K=n_in + 1, family="fc", store="fp32",
                act=act, v=v.reshape(-1))]


def _spec_channel_scale(a, st):
    dt = _vec_dtype(a)
    B, S_, C_ = a["B"], a["S"], a["C"]
    x = cl(st, a["x"], B * S_, a["cstride"], C_, dt, inplace=True)
    return [x, flat(st, a["gate"], B * C_, torch.float32)], [x]


def _ref_channel_scale(a, R, W, prec):
    B, S_, C_ = a["B"], a["S"], a["C"]
    x = R[0].to(f64).view(B, S_, C_)
    ref = (x * R[1].to(f64).view(B, 1, C_)).reshape(B * S_, C_)
    return [Out(idx=0, ref=ref, S=ref.abs() * 2.0 ** -24, K=1, family=None, store=STORE[a["dtype"]], act="none")]


def _spec_cl_transpose(a, st):
    dt = _vec_dtype(a)
    B, P, C_, cs, ldo, ob = a["B"], a["P"], a["C"], a["cstride"], a["ldo"], a["out_bstride"]
    es = torch.empty(0, dtype=dt).element_size()
    k, off = st.place(a["in"] + a["coff"] * es)
    reads = [Reg(k, off, (B * P, C_), (cs, 1), dt, win=(C_, cs))]
    k, off = st.place(a["out"])
    return reads, [Reg(k, off, (B, C_, P), (ob, ldo, 1), dt)]


def _ref_cl_transpose(a, R, W, prec):
    B, P, C_ = a["B"], a["P"], a["C"]
    return [Out(idx=0, exact=R[0].view(B, P, C_).permute(0, 2, 1))]


def _spec_copy(a, st):
    dt = _vec_dtype(a)
    es = torch.empty(0, dtype=dt).element_size()
    n, C_ = a["positions"], a["C"]
    return ([cl(st, a["in"] + a["in_coff"] * es, n, a["in_cstride"], C_, dt)],
            [cl(st, a["out"] + a["out_coff"] * es, n, a["out_cstride"], C_, dt)])


def _ref_copy(a, R, W, prec):
    return [Out(idx=0, exact=R[0])]


def _spec_vview(a, st):
    dt = _vec_dtype(a)
    B, h, w, Cw, dh, dw = a["B"], a["h"], a["w"], _r8(a["C"]), a["dh"], a["dw"]
    ds = a.get("depth_stride", 0)
    nd = dh * dw if ds == 0 else (B - 1) * ds + dh * dw
    return ([cl(st, a["in"], B * h * w, a["cs_in"], Cw, dt), flat(st, a["depth"], nd, torch.float32)],
            [cl(st, a["out"], B * h * w, a["cs_out"], Cw, dt)])


def _ref_vview(a, R, W, prec):
    B, h, w, Cw, dh, dw = a["B"], a["h"], a["w"], _r8(a["C"]), a["dh"], a["dw"]
    ds = a.get("depth_stride", 0)
    x = R[0].to(f64).view(B, h, w, Cw)
    outs, Ss = [], []
    for b in range(B):
        d = R[1][b * ds:b * ds + dh * dw].to(f64).view(dh, dw)
        o, s = virtual_view_ref(x[b], d, a["bf_scale"])
        outs.append(o)
        Ss.append(s)
    sh = (B * h * w, Cw)
    return [Out(idx=0, ref=torch.stack(outs).reshape(sh), S=torch.stack(Ss).reshape(sh), K=4, family="vview",
                store=STORE[a["dtype"]], act="none")]


_VV = ["in", "out", "depth", "dtype", "B", "h", "w", "C", "cs_in", "cs_out", "dh", "dw", "bf_scale"]
_DW = ["in", "w", "bias", "out", "pool", "dtype", "B", "H", "W", "OH", "OW", "C", "cs_in", "cs_out", "K", "stride",
       "pad_top", "pad_left", "act", "stream"]
SPECS = {
    "occd_dwconv2d_tiled_fwd": types.SimpleNamespace(args=_DW, regions=_spec_dwconv, ref=_ref_dwconv),
    "occd_se_gate_fold_fwd": types.SimpleNamespace(
        args=["pool", "inv_hw", "w1", "b1", "w2t", "b2", "hidden", "master", "wout", "wdtype", "B", "C", "R", "rows",
              "Kpad", "stream"], regions=_spec_se_fold, ref=_ref_se_fold),
    "occd_upsample_bilinear_ac": types.SimpleNamespace(
        args=["in", "out", "dtype", "B", "h", "w", "OH", "OW", "C", "cs_in", "in_off", "cs_out", "out_off", "stream"],
        regions=_spec_bilinear, ref=_ref_bilinear),
    "occd_upsample_tapsum_ac": types.SimpleNamespace(
        args=["y", "pre", "out", "dtype", "B", "h", "w", "OH", "OW", "C", "cs_y", "y_off", "tap_stride", "cs_pre",
              "pre_off", "cs_out", "out_off", "act", "stream"], regions=_spec_tapsum, ref=_ref_tapsum),
    "occd_sfa_lift_fwd": types.SimpleNamespace(args=["p", "stream"], regions=_spec_lift, ref=_ref_lift),
    "occd_frustum_sample_window_fwd": types.SimpleNamespace(
        args=["depth", "cams", "V", "Dn", "h", "w", "X", "Y", "Z", "x0", "Xl", "img_w", "img_h", "dmin", "dmax",
              "mean_mode", "out", "perm_xzy", "stream"], regions=_spec_prior, ref=_ref_prior),
    "occd_grid_sample_prior_window_fwd": types.SimpleNamespace(
        args=["depth", "grids", "V", "Dn", "h", "w", "X", "Y", "Z", "x0", "Xl", "mean_mode", "out", "perm_xzy",
              "stream"], regions=_spec_prior, ref=_ref_prior),
    "occd_softmax_planar": types.SimpleNamespace(args=["in", "out", "B", "C", "S", "stream"], regions=_spec_softmax,
                                                 ref=_ref_softmax),
    "occd_softmax_planar_to_cl": types.SimpleNamespace(
        args=["in", "out", "dtype", "B", "C", "S", "cstride", "coff", "stream"], regions=_spec_softmax_cl,
        ref=_ref_softmax_cl),
    "occd_fc_fwd": types.SimpleNamespace(args=["in", "w", "bias", "out", "B", "n_in", "n_out", "act", "stream"],
                                         regions=_spec_fc, ref=_ref_fc),
    "occd_channel_scale": types.SimpleNamespace(args=["x", "gate", "dtype", "B", "S", "C", "cstride", "stream"],
                                                regions=_spec_channel_scale, ref=_ref_channel_scale),
    "occd_cl_transpose": types.SimpleNamespace(
        args=["in", "out", "dtype", "B", "P", "C", "cstride", "coff", "ldo", "out_bstride", "stream"],
        regions=_spec_cl_transpose, ref=_ref_cl_transpose),
    "occd_copy_channels": types.SimpleNamespace(
        args=["in", "out", "dtype", "positions", "C", "in_cstride", "in_coff", "out_cstride", "out_coff", "stream"],
        regions=_spec_copy, ref=_ref_copy),
    "occd_virtual_view_fwd": types.SimpleNamespace(args=_VV + ["stream"], regions=_spec_vview, ref=_ref_vview),
    "occd_virtual_view_items_fwd": types.SimpleNamespace(args=_VV + ["depth_stride", "stream"], regions=_spec_vview,
                                                         ref=_ref_vview),
}


# ---------------------------------------------------------------------------------------------------------------
# one launch: snapshot, poison, run, compare, restore
def _byte_view(s):
    return torch.empty(0, dtype=torch.uint8, device=s.device).set_(s, 0, (s.nbytes(),), (1,))


def _poison_value(dtype):
    return float("nan") if dtype.is_floating_point else None


class Launch:
    """one recorded launch over a plan's storages: its regions, and the state of every storage it reaches"""

    def __init__(self, rec, st):
        self.rec, self.st = rec, st
        self.name = rec[0]
        self.a = named(rec)
        self.spec = SPECS[self.name]
        self.reads, self.writes = self.spec.regions(self.a, st)
        self.keys = sorted({r.key for r in self.reads + self.writes})
        self.storages = {k: st.by_key[k] for k in self.keys}

    def snapshot(self):
        return {k: _byte_view(s).clone() for k, s in self.storages.items()}

    def restore(self, snap):
        for k, s in self.storages.items():
            _byte_view(s).copy_(snap[k])

    def poison(self):
        """NaN into the output regions (not the in-place ones) and into the channels outside each channels-last input
        window at the rows the launch reads (where no other input or output of the launch lies)"""
        keep = {k: torch.zeros(s.nbytes(), dtype=torch.uint8, device=s.device) for k, s in self.storages.items()}
        for r in self.reads + self.writes:
            r.byte_mask(keep[r.key])
        for r in self.writes:
            if not r.inplace and _poison_value(r.dtype) is not None:
                r.view(self.storages).fill_(float("nan"))
        for r in self.reads:
            if r.win is None or not r.dtype.is_floating_point:
                continue
            Cw, cs = r.win
            if cs == Cw:
                continue
            es = torch.empty(0, dtype=r.dtype).element_size()
            nb = self.storages[r.key].nbytes()
            rows = r.shape[0]
            # rows [p + i cs + Cw, p + (i + 1) cs), clipped to the storage
            n_full = min(rows, (nb - r.off) // (cs * es))
            if n_full <= 0:
                continue
            out = Reg(r.key, r.off + Cw * es, (n_full, cs - Cw), (cs, 1), r.dtype)
            v = out.view(self.storages)
            m = torch.zeros(nb, dtype=torch.uint8, device=v.device)
            out.byte_mask(m)
            m &= 1 - keep[r.key]
            bad = m.view(-1)[r.off + Cw * es:].as_strided((n_full, cs - Cw), (cs * es, es))
            v.masked_fill_(bad.bool(), float("nan"))

    def reads_of(self, storages=None):
        return [r.view(storages or self.storages) for r in self.reads]


def replay(rec, st, stream, lib_sync=None):
    """-> (fails, stats, launch) after running `rec` alone on `stream` (GPU)"""
    L = Launch(rec, st)
    orig = L.snapshot()
    L.poison()
    before = L.snapshot()
    ins = [x.clone() for x in L.reads_of()]
    pool_before = None
    if L.name == "occd_dwconv2d_tiled_fwd" and L.a["pool"]:
        pool_before = L.writes[1].view(L.storages).clone()
    rc = call(rec, stream)
    torch.cuda.synchronize()
    if rc != 0:
        L.restore(orig)
        return ["%s returned %d" % (L.name, rc)], {}, L
    outs = [w.view(L.storages) for w in L.writes]
    prec = "tf32" if L.a.get("dtype", L.a.get("wdtype", 0)) == 0 else "bf16"
    refs = L.spec.ref(L.a, ins, outs, prec)
    fails, stats = compare(L, refs, outs, prec, pool_before)
    fails += moved(L, before)
    L.restore(orig)
    return fails, stats, L


def moved(L, before):
    """bytes outside the declared output regions that differ from their state before the launch"""
    fails = []
    for k, s in L.storages.items():
        allowed = torch.zeros(s.nbytes(), dtype=torch.uint8, device=s.device)
        for w in L.writes:
            if w.key == k:
                w.byte_mask(allowed)
        diff = (_byte_view(s) != before[k]) & (allowed == 0)
        if bool(diff.any()):
            at = diff.nonzero()
            fails.append("moved outside the output regions: %d byte(s) of a %d-byte storage, first at byte %d"
                         % (at.shape[0], s.nbytes(), int(at[0])))
    return fails


def family_constant(family, prec):
    return C_ACC[family][prec]


def compare(L, refs, outs, prec, pool_before=None):
    fails, stats = [], {}
    for o in refs:
        got = outs[o.idx]
        what = "%s output %d" % (L.name, o.idx)
        if getattr(o, "zero", False):
            if bool((got != 0).any()):
                fails.append("%s: not zero afterwards" % what)
            continue
        if getattr(o, "exact", None) is not None:
            if not torch.equal(CR._bits(got.contiguous()), CR._bits(o.exact.contiguous())):
                n = int((CR._bits(got.contiguous()) != CR._bits(o.exact.contiguous())).sum())
                fails.append("%s: %d element(s) differ from the data they move" % (what, n))
            continue
        if getattr(o, "pool", False):
            f, s = check_pool(got, pool_before, L.writes[0].view(L.storages), o, prec)
            fails += f
            CR._merge(stats, s)
            continue
        bad, excess, s = check(got.to(f64), o, prec)
        CR._merge(stats, s)
        if bool(bad.any()):
            i = int(torch.where(bad, excess, torch.full_like(excess, -1.0)).flatten().argmax())
            fails.append("%s: %d element(s) beyond the bound; worst flat index %d: got %r, float64 %r, %.3g beyond"
                         % (what, int(bad.sum()), i, float(got.flatten()[i]), float(o.ref.flatten()[i]),
                            float(excess.flatten()[i])))
        if o.store == "tf32":
            nt = (CR._bits(got.contiguous()) & 0x1FFF) != 0
            if bool(nt.any()):
                fails.append("%s: a stored element is not a TF32 value" % what)
    return fails, stats


def check(got, o, prec, c=None):
    """conv_replay.check with the family's constant -> (bad, excess, {family: observed ratio})"""
    ref, S, K = o.ref, o.S, o.K
    if o.family is None:                  # one rounding of one fp32 result: S is that rounding's bound
        err = (got - ref).abs()
        bound = 0.5 * ulp_store(ref.abs() + S, o.store) + S
        return ~(err <= bound), err - bound, {}
    c = family_constant(o.family, prec) if c is None else c
    a_act = getattr(o, "a_act", None)
    if a_act is None and o.act == "silu":
        a_act = A_ACT[prec].get("silu", 0.0)
    bad, excess, st = CR.check(got, ref, S, K, o.store, prec, o.act, getattr(o, "v", None), None, c_acc=c,
                               a_act=a_act or 0.0)
    key = o.family + ("" if o.act not in ("silu", "sigmoid") else "." + o.act)
    return bad, excess, {key: v for v in st.values()}


def pool_blocks(OH, OW):
    """blocks of the tiled depthwise kernel that add into one (image, channel) sum: tiles of at least 8 rows x 16
    columns (csrc/dwconv_tiled.cuh)"""
    return -(-OH // 8) * -(-OW // 16)


def check_pool(pool_after, pool_before, out, o, prec, c=None):
    """pool_after - pool_before == 2^24 sum of the stored outputs, within 1/2 per contributing block plus the fp32
    partial sums' rounding"""
    c = C_ACC["pool"][prec] if c is None else c
    B, C_, OH, OW = o.B, o.C, o.OH, o.OW
    y = out[:, :C_].to(f64).view(B, OH * OW, C_)
    want = y.sum(1) * 2.0 ** 24
    S = y.abs().sum(1) * 2.0 ** 24
    got = (pool_after - pool_before).to(f64)
    half = 0.5 * pool_blocks(OH, OW)
    err = (got - want).abs()
    bound = half + c * (OH * OW) ** 0.5 * S
    fails = []
    if bool((~(err <= bound)).any()):
        i = int((err - bound).flatten().argmax())
        fails.append("squeeze pool: %d sum(s) beyond the bound; worst (b, c) = %s: got %d, 2^24 sum of the stored "
                     "outputs %.1f" % (int((~(err <= bound)).sum()), divmod(i, C_), int(got.flatten()[i]),
                                       float(want.flatten()[i])))
    pos = S > 0
    stats = {}
    if bool(pos.any()):
        stats["pool"] = float(((err - half)[pos] / S[pos]).max()) / (OH * OW) ** 0.5
    return fails, stats


def dw_menu(a, n_sms):
    """(cvb, TH, PX) of the tiled depthwise kernel for a recorded launch (dwt::choose, csrc/dwconv_tiled.cuh)"""
    f32 = a["dtype"] == 0
    C_, S = a["C"], a["stride"]
    cvb = 4 if (C_ < 64 or f32) else 8
    if cvb == 4:
        th = 16
    elif S == 2:
        th = 8
    else:
        th = 16 if a["B"] * -(-a["OH"] // 16) * -(-a["OW"] // 16) * -(-C_ // 64) >= 4 * n_sms else 8
    px = 8 if (cvb == 4 and f32 and S == 1) else 4
    return cvb, th, px


def lift_menu(p):
    """(dtype, V, NV, G) of the lift kernel (launch_nv, csrc/sfa_lift.cu)"""
    dt = "f32" if p.feat_dtype == 0 else "bf16"
    vecs = -(-p.C // (4 if dt == "f32" else 8))
    if vecs <= 4:
        return dt, p.n_views, 1, 4
    nv = 2 if dt == "bf16" else 4
    lanes = (4, 8, 16, 32) if dt == "bf16" else (2, 4, 8, 16)
    for lim, g in zip((8, 16, 32, 64), lanes):
        if vecs <= lim:
            return dt, p.n_views, nv, g
    return dt, p.n_views, None, None


@contextlib.contextmanager
def no_recorder():
    from occdepth_b200 import _lib
    saved = getattr(_lib._RECORDING, "recorder", None)
    _lib._RECORDING.recorder = None
    try:
        yield
    finally:
        _lib._RECORDING.recorder = saved

