"""Per-launch convolution parity: one planned `engine.ConvOp` replayed alone, in place, against float64.

Shared by tests/test_conv_replay_host.py and tests/test_gpu_conv_replay.py (a plain helper, imported like gpu_cases).

  signature(op)   hashable record of everything that can change what the kernel does; equal signatures are the same
                  launch on different data
  fill(op, seed)  seeded values, rounded to the storage type, into the WHOLE storage of every buffer the op can reach
  Snapshot(op)    copies of those storages, and the descriptor as plain numbers
  reference(snap) the operation in float64, written from the ABI's description of occd_conv_desc
                  (include/occdepth_b200.h): tap reads with zero outside the buffer and margin data inside it, tap
                  groups, per-image weights, v = acc + bias + res1 (+ res2), out1 = v, out0 = act(v) (+ res2 when
                  post); and S, the same sum with every term's absolute value -- the scale of the accumulation error
  check(...)      element-wise:  |got - ref| <= 1/2 ulp_store(|ref| + d) + d,   d = L(act) C_ACC sqrt(K) S + A_ACT a(v)
                  ulp_store is the spacing of the storage type (TF32: 10 mantissa bits, bf16: 7, fp32 for out0_exact
                  and planar out1), taken at the largest magnitude the device's fp32 value can have; K is the number
                  of products in one output's sum (source channels over the taps of its group): over the sweep the
                  error of the fp32 accumulation grows as sqrt(K) from K = 6 to K = 64800, so one constant per
                  precision in front of sqrt(K) S stays sharp for the short sums, which a constant sized for the
                  longest could not; L = 1.1 for SiLU (its largest slope), else 1; a(v) = |v| for SiLU, 1 for the
                  sigmoid, 0 for the exact activations
  check_op(...)   every output of the launch through check(); TF32 bit pattern of tf32 stores; the class map, where
                  a differing class needs a float64 gap within the accumulation bound; the float16 confidence (out1
                  mode 4) and probabilities (mode 5) through check_prob(), taken at the class the map holds, and in
                  mode 5 the map's class holding the largest probability bit for bit; and NOTHING ELSE MOVES: every
                  byte of every reachable storage equals the snapshot except channels [coff, coff + roundup(Cout, 8))
                  of the output window at the launch's output positions (planar out1: [out1_coff, out1_coff + Cout);
                  class modes: the uint16 map [B P] (P positions), then [B P] of confidence or [B Cout P] of
                  probabilities at out1[B P + (b Cout + n) P + s]).
                  The pad channels [Cout, roundup(Cout, 8)) are checked like any other: they hold what the epilogue
                  makes of a zero accumulator (zero without activation and residual -- DESIGN.md section 3).

The constants are at most twice the largest ratio seen over the sweep of tests/test_gpu_conv_replay.py (all six shipped
configurations, both precisions, forward + class-map + two slab rank plans: 1276 distinct launches) on an NVIDIA H100
80GB HBM3 (power limit 700 W), which found no failing launch:

  largest (|got - ref| - 1/2 ulp) / (sqrt(K) S), exact activations:   tf32 3.78e-8   bf16 3.05e-8
  largest (|got - ref| - 1/2 ulp - L C_ACC sqrt(K) S) / a(v):         bf16 SiLU (tanh.approx) 3.1e-6;
      below zero for the tf32 SiLU and both sigmoids (__expf / __fdividef): the accumulation term already covers
      them, so they get no term of their own

The confidence and probabilities (check_prob):  |got - p| <= 1/2 ulp_f16(p + d) + d,  d = p (delta_c + sum_j p_j
delta_j) + A_SM p, with p the float64 softmax of v over the Cout classes and delta_j = C_ACC sqrt(K) S_j the bound on
class value j (an fp32 sum plus bias and residuals, never rounded to the storage type).  A_SM would cover expf, the fp32
sum over the classes and the division; the largest (|got - p| - 1/2 ulp_f16 - d + A_SM p) / p over both sweeps is below
zero (shipped: tf32 -4.6e-7, bf16 -3.3e-7; menu: tf32 -7.9e-6, bf16 -8.7e-6), so, like the exact activations, they
get no term of their own: A_SM = 0.
"""
import types
import zlib

import torch

from occdepth_b200 import _lib

ACT_NAME = {_lib.ACT_NONE: "none", _lib.ACT_RELU: "relu", _lib.ACT_LEAKY: "leaky", _lib.ACT_SILU: "silu",
            _lib.ACT_SIGMOID: "sigmoid"}
IMPL_NAME = {_lib.CONV_IMPL_TC: "tc", _lib.CONV_IMPL_SIMT: "simt", _lib.CONV_IMPL_HALO: "halo",
             _lib.CONV_IMPL_HALOX: "halox", _lib.CONV_IMPL_TCX: "tcx"}
MANT = {"tf32": 10, "bf16": 7, "fp32": 23, "f16": 10}          # explicit mantissa bits of the storage types
EMIN = {"f16": -14}                                            # smallest normal exponent (default: fp32's -126)

C_ACC = {"tf32": 6.0e-8, "bf16": 5.0e-8}
A_ACT = {"tf32": dict(), "bf16": dict(silu=5.0e-6)}
ACT_SLOPE = dict(silu=1.1)
A_SM = {"tf32": 0.0, "bf16": 0.0}
OBSERVED = {}        # sweep -> precision -> observed maxima (check / check_prob stats) of the GPU sweeps of a session


def _ceil_div(a, b):
    return -((-a) // b)


def precision_of(t):
    return "tf32" if t.dtype == torch.float32 else "bf16"


# ---------------------------------------------------------------------------------------------------------------
# the descriptor as plain numbers
def desc_fields(op):
    d = op.desc
    n = d.n_src
    D = dict(dtype=d.dtype, B=d.B, ID=d.ID, IH=d.IH, IW=d.IW, src_d0=d.src_d0, stride=tuple(d.stride),
             src_C=tuple(d.src_C[:n]), src_cstride=tuple(d.src_cstride[:n]), src_coff=tuple(d.src_coff[:n]),
             taps=tuple((t.src, t.dz, t.dy, t.dx) for t in d.taps[:d.n_taps]),
             Cout=d.Cout, Cout_pad=d.Cout_pad, Kpad=d.Kpad, weight_per_image=d.weight_per_image,
             O=(d.OD, d.OH, d.OW), omul=tuple(d.omul), Of=(d.ODf, d.OHf, d.OWf), act=ACT_NAME[d.act],
             out0=bool(d.out0), out0_cstride=d.out0_cstride, out0_coff=d.out0_coff, out0_exact=d.out0_exact,
             res1=bool(d.res1), res1_cstride=d.res1_cstride, res1_coff=d.res1_coff,
             res2=bool(d.res2), res2_cstride=d.res2_cstride, res2_coff=d.res2_coff, res2_post=d.res2_post,
             out1_mode=d.out1_mode, out1_cstride=d.out1_cstride, out1_coff=d.out1_coff, out1_C=d.out1_C)
    if d.n_groups > 1:      # group g: taps [tap0[g], tap0[g + 1]) written at o * omul + group_oadd[g]
        D["groups"] = tuple((d.group_tap0[g], d.group_tap0[g + 1], tuple(d.group_oadd[g])) for g in range(d.n_groups))
    else:
        D["groups"] = ((0, d.n_taps, tuple(d.oadd)),)
    return D


def signature(op):
    """hashable; the kernel-choice fields (kernel, tile box, N tile, K chunk, stages, grid, schedule) are absent for
    the SIMT flavour, the only one that plans without a driver"""
    D = desc_fields(op)
    kernel = None
    if op.impl != _lib.CONV_IMPL_SIMT:
        kernel = (IMPL_NAME[op.impl],) + tuple(sorted(op.info().items()))
    return tuple(sorted(D.items())) + (("kernel", kernel), ("lut", op.lut is not None))


def seed_of(sig):
    return zlib.crc32(repr(sig).encode())


# ---------------------------------------------------------------------------------------------------------------
# storage types
def quantize(x, store, mode=None):
    """float64 -> nearest value of the storage type, as float64.  mode: 'away' (cvt.rna, the TF32 stores), 'even'
    (bf16 / fp32 stores) or 'trunc' (what a store must NOT do); default: the type's own rounding"""
    mode = mode or ("away" if store == "tf32" else "even")
    m, e = torch.frexp(x)
    k = float(2 ** (MANT[store] + 1))
    s = m * k
    if mode == "away":
        q = torch.sign(s) * torch.floor(s.abs() + 0.5)
    elif mode == "even":
        q = torch.round(s)
    else:
        q = torch.trunc(s)
    return torch.ldexp(q / k, e)


def ulp_store(x, store):
    """spacing of the storage type at magnitude x (float64, >= 0); 0 at 0"""
    _, e = torch.frexp(x)
    e = (e - 1).clamp_min(EMIN.get(store, -126)) - MANT[store]
    return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e), torch.zeros_like(x))


def to_store(x, dtype):
    """fp32 -> the storage dtype, rounded as the layout kernels round"""
    if dtype == torch.bfloat16:
        return x.to(torch.bfloat16)
    return ((x.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


def _whole(t):
    """the whole storage behind t as a flat tensor of t's dtype"""
    st = t.untyped_storage()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(st, 0, (st.nbytes() // t.element_size(),))


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


# ---------------------------------------------------------------------------------------------------------------
def reach(op):
    """[(role, tensor)] of every buffer the launch can touch, sources first"""
    r = [("src", s.buf) for s in op.srcs]
    for role in ("out0", "res1", "res2"):
        cl = getattr(op, role)
        if cl is not None:
            r.append((role, cl.buf))
    if op.out1 is not None:
        r.append(("out1_" + op.out1_mode, op.out1.buf if op.out1_mode == "cl" else op.out1))
    return r + [("weight", op.weight), ("bias", op.bias)]


def fill(op, seed):
    """seeded values into the whole storage of every activation buffer the op reaches (a storage shared by a source
    and an output is filled once), rounded to its type; a run-time weight buffer gets seeded weights with the ABI's
    zero padding.  Sources get a seeded choice of randn or relu(randn) + 0.1 (a post-activation map)."""
    D = desc_fields(op)
    dev = op.bias.device
    g = torch.Generator(device=dev).manual_seed(seed)
    positive = bool(seed & 1)
    done = set()
    for role, t in reach(op):
        if role in ("weight", "bias"):
            continue
        key = t.untyped_storage().data_ptr()
        if key in done:
            continue
        done.add(key)
        w = _whole(t)
        if t.dtype == torch.uint16:
            _bits(w).fill_(-1)
            continue
        x = torch.randn(w.numel(), generator=g, device=dev)
        if role == "src" and positive:
            x = torch.relu(x) + 0.1
        w.copy_(x if role == "out1_planar" else to_store(x, t.dtype))
    if op.weight_runtime:
        nt = len(D["taps"])
        W = op.weight.view(-1, D["Cout_pad"], D["Kpad"])
        W.zero_()
        ktot = sum(D["src_C"][t[0]] for t in D["taps"])
        for i in range(W.shape[0]):
            c = D["src_C"][D["taps"][i % nt][0]]
            x = torch.randn(D["Cout"], c, generator=g, device=dev) / ktot ** 0.5
            W[i, :D["Cout"], :c] = to_store(x, W.dtype)


class Snapshot:
    """the launch's descriptor numbers and a copy of every storage it can reach, taken before it runs"""

    def __init__(self, op):
        self.D = desc_fields(op)
        # products in one output's sum: the source channels over the taps of its (largest) group
        self.K = max(sum(self.D["src_C"][t[0]] for t in self.D["taps"][t0:t1]) for t0, t1, _ in self.D["groups"])
        self.precision = precision_of(op.srcs[0].buf)
        self.lut = op.lut
        self.store = {}
        for _, t in reach(op):
            key = t.untyped_storage().data_ptr()
            if key not in self.store:
                self.store[key] = _whole(t).clone()
        self.srcs = [self.of(s.buf) for s in op.srcs]
        self.res1 = None if op.res1 is None else self.of(op.res1.interior())
        self.res2 = None if op.res2 is None else self.of(op.res2.interior())
        self.weight, self.bias = self.of(op.weight), self.of(op.bias)

    def of(self, t):
        """the snapshot's copy of tensor t"""
        return self.store[t.untyped_storage().data_ptr()].as_strided(t.shape, t.stride(), t.storage_offset())


def _valid(base, off, s, I, O, lo, hi):
    """output range [a, b) within [lo, hi) whose input coordinate base + o * s + off lies in [0, I)"""
    a = max(lo, _ceil_div(-(base + off), s))
    b = min(hi, (I - 1 - base - off) // s + 1, O)
    return a, b


def reference(snap, chunk_bytes=1 << 28):
    """-> namespace(v, S, out0, mask): float64 [B, ODf, OHf, OWf, Cw] on the full output grid over the Cw =
    roundup(Cout, 8) channels the launch stores (v: pre-activation = out1; out0: None without an out0), and the bool
    mask [ODf, OHf, OWf] of the positions the launch writes.  Unwritten positions hold zeros."""
    D = snap.D
    B, Cout = D["B"], D["Cout"]
    Cw = (Cout + 7) // 8 * 8
    O, Of, st, om = D["O"], D["Of"], D["stride"], D["omul"]
    I = (D["ID"], D["IH"], D["IW"])
    base = (D["src_d0"], 0, 0)
    dev = snap.bias.device
    f64 = torch.float64
    X = [s[..., c0:c0 + c] for s, c0, c in zip(snap.srcs, D["src_coff"], D["src_C"])]
    nt = len(D["taps"])
    W = snap.weight.view(-1, D["Cout_pad"], D["Kpad"])
    bias = snap.bias[:Cw].to(f64)
    v = torch.zeros((B,) + Of + (Cw,), dtype=f64, device=dev)
    S = torch.zeros_like(v)
    out0 = torch.zeros_like(v) if D["out0"] else None
    mask = torch.zeros(Of, dtype=torch.bool, device=dev)
    ax = 0 if O[0] > 1 else 1
    per_row = B * (O[0] * O[1] * O[2] // O[ax]) * max(max(D["src_C"]), Cw) * 8
    rows = max(1, chunk_bytes // per_row)
    for (t0, t1, oadd) in D["groups"]:
        for c0 in range(0, O[ax], rows):
            lo = [0, 0, 0]
            hi = list(O)
            lo[ax], hi[ax] = c0, min(O[ax], c0 + rows)
            n = [hi[i] - lo[i] for i in range(3)]
            acc = torch.zeros([B] + n + [Cw], dtype=f64, device=dev)
            sab = torch.zeros_like(acc)
            for ti in range(t0, t1):
                si, dz, dy, dx = D["taps"][ti]
                r = [_valid(base[i], (dz, dy, dx)[i], st[i], I[i], O[i], lo[i], hi[i]) for i in range(3)]
                if any(a >= b for a, b in r):
                    continue
                isl = tuple(slice(base[i] + r[i][0] * st[i] + (dz, dy, dx)[i],
                                  base[i] + (r[i][1] - 1) * st[i] + (dz, dy, dx)[i] + 1, st[i]) for i in range(3))
                osl = tuple(slice(r[i][0] - lo[i], r[i][1] - lo[i]) for i in range(3))
                x = X[si][(slice(None),) + isl].to(f64)
                C_ = x.shape[-1]
                for b in (range(B) if D["weight_per_image"] else [None]):
                    w = W[ti if b is None else b * nt + ti, :Cw, :C_].to(f64).t()
                    bs = slice(None) if b is None else slice(b, b + 1)
                    acc[(bs,) + osl] += x[bs] @ w
                    sab[(bs,) + osl] += x[bs].abs() @ w.abs()
            fsl = (slice(None),) + tuple(slice(oadd[i] + lo[i] * om[i], oadd[i] + (hi[i] - 1) * om[i] + 1, om[i])
                                         for i in range(3))
            vv = acc + bias
            ss = sab + bias.abs()
            r2 = None
            if snap.res1 is not None:
                r1 = snap.res1[fsl][..., D["res1_coff"]:D["res1_coff"] + Cw].to(f64)
                vv += r1
                ss += r1.abs()
            if snap.res2 is not None:
                r2 = snap.res2[fsl][..., D["res2_coff"]:D["res2_coff"] + Cw].to(f64)
                ss += r2.abs()
                if not D["res2_post"]:
                    vv += r2
            v[fsl], S[fsl] = vv, ss
            mask[fsl[1:]] = True
            if out0 is not None:
                y = activation(vv, D["act"])
                if r2 is not None and D["res2_post"]:
                    y = y + r2
                out0[fsl] = y
    return types.SimpleNamespace(v=v, S=S, out0=out0, mask=mask, Cw=Cw)


def activation(v, act):
    if act == "relu":
        return torch.relu(v)
    if act == "leaky":
        return torch.where(v > 0, v, 0.01 * v)
    if act == "silu":
        return v * torch.sigmoid(v)
    if act == "sigmoid":
        return torch.sigmoid(v)
    assert act == "none", act
    return v


# ---------------------------------------------------------------------------------------------------------------
def check(got, ref, S, K, store, precision, act="none", v=None, where=None, c_acc=None, a_act=None):
    """element-wise bound (module docstring).  got / ref / S / v: float64 of one shape; K: products per sum; store:
    type of the stored value ('tf32' | 'bf16' | 'fp32'); act: the activation between v and ref ('none' for out1);
    where: bool mask (broadcastable) of the elements that count, default all.
    -> (bad: bool tensor, excess: err - bound, stats: dict(acc=..., silu=..., sigmoid=...) of observed maxima)"""
    c = (C_ACC[precision] if c_acc is None else c_acc) * K ** 0.5
    d = ACT_SLOPE.get(act, 1.0) * c * S
    scale = None
    if act in ("silu", "sigmoid"):
        scale = v.abs() if act == "silu" else torch.ones_like(S)
        d = d + (A_ACT[precision].get(act, 0.0) if a_act is None else a_act) * scale
    err = (got - ref).abs()
    bound = 0.5 * ulp_store(ref.abs() + d, store) + d
    bad = ~(err <= bound)                      # a NaN fails
    if where is not None:
        bad = bad & where
    e = err - 0.5 * ulp_store(torch.maximum(ref.abs(), got.abs()), store)
    stats = {}
    if scale is None:
        pos = (S > 0) if where is None else ((S > 0) & where)
        if bool(pos.any()):
            stats["acc"] = float((e[pos] / S[pos]).max()) / K ** 0.5
    else:
        e = e - ACT_SLOPE.get(act, 1.0) * c * S
        pos = (scale > 0) if where is None else ((scale > 0) & where)
        if bool(pos.any()):
            stats[act] = float((e[pos] / scale[pos]).max())
    return bad, err - bound, stats


CLASS_OUT1 = (_lib.OUT1_CLASS_U16, _lib.OUT1_CLASS_U16_CONF, _lib.OUT1_CLASS_U16_PROBS)


def _merge(stats, new):
    for k, val in new.items():
        stats[k] = max(stats.get(k, val), val)


def _window(cl, coff, Cw):
    return cl.interior()[..., coff:coff + Cw]


def check_op(op, snap, R, info=None):
    """-> (failures: list of report strings, stats).  info: op.info() of a tensor-core plan, for the tile coordinates
    of a failure report."""
    D = snap.D
    prec = snap.precision
    Cout, Cw = D["Cout"], R.Cw
    fails, stats = [], {}
    f64 = torch.float64
    m = R.mask
    full = bool(m.all())
    restored = {k: _whole_of(op, k).clone() for k in snap.store}     # live copies; output windows get put back

    def view(t):
        return restored[t.untyped_storage().data_ptr()].as_strided(t.shape, t.stride(), t.storage_offset())

    def put_back(t, csl):
        """overwrite the launch's output window of live copy `t` [B, D, H, W, C] with the snapshot's"""
        a, b = view(t), snap.of(t)
        if full:
            a[..., csl] = b[..., csl]
        else:
            a[:, m, csl] = b[:, m, csl]

    where = None if full else m[None, :, :, :, None]

    def not_tf32(got):
        x = (_bits(got.contiguous()) & 0x1FFF) != 0
        return bool((x if full else x & where).any())

    def elementwise(what, got, ref, store, act):
        bad, excess, st = check(got.to(f64), ref, R.S, snap.K, store, prec, act, R.v, where)
        _merge(stats, st)
        if bool(bad.any()):
            fails.append(describe(what, D, bad, excess, got, ref, info))

    if D["out0"]:
        cl = op.out0
        got = _window(cl, D["out0_coff"], Cw)
        store = "fp32" if (D["out0_exact"] and prec == "tf32") else prec
        elementwise("out0", got, R.out0, store, D["act"])
        if store == "tf32" and not_tf32(got):
            fails.append("out0: a stored element is not a TF32 value (low 13 mantissa bits set)")
        put_back(cl.interior(), slice(D["out0_coff"], D["out0_coff"] + Cw))
    if D["out1_mode"] == _lib.OUT1_CL:
        cl = op.out1
        got = _window(cl, D["out1_coff"], Cw)
        elementwise("out1", got, R.v, prec, "none")
        if prec == "tf32" and not_tf32(got):
            fails.append("out1: a stored element is not a TF32 value (low 13 mantissa bits set)")
        put_back(cl.interior(), slice(D["out1_coff"], D["out1_coff"] + Cw))
    elif D["out1_mode"] == _lib.OUT1_F32_PLANAR:
        c0 = D["out1_coff"]
        got = op.out1[:, c0:c0 + Cout].permute(0, 2, 3, 4, 1)
        bad, excess, st = check(got.to(f64), R.v[..., :Cout], R.S[..., :Cout], snap.K, "fp32", prec, "none", None,
                                where)
        _merge(stats, st)
        if bool(bad.any()):
            fails.append(describe("out1 (planar)", D, bad, excess, got, R.v[..., :Cout], info))
        put_back(op.out1.permute(0, 2, 3, 4, 1), slice(c0, c0 + Cout))
    elif D["out1_mode"] in CLASS_OUT1:
        assert full                 # a class map needs no tap groups, and no planned one is written on a sub-grid
        mode = D["out1_mode"]
        B = D["B"]
        u16 = op.out1.reshape(-1, *D["Of"])          # [B] map rows, then [B] confidence or [B * Cout] probability rows
        c_acc = C_ACC[prec] * snap.K ** 0.5
        got = _bits(u16[:B]).to(torch.int64) & 0xFFFF
        msg = check_classes(got, R.v[..., :Cout], R.S[..., :Cout], snap.lut, c_acc)
        if msg:
            fails.append(msg)
        if mode != _lib.OUT1_CLASS_U16:
            P, d = softmax_bound(R.v[..., :Cout], R.S[..., :Cout], c_acc)
            k = chosen_class(got, R.v[..., :Cout], snap.lut)
            if mode == _lib.OUT1_CLASS_U16_CONF:
                what, half = "confidence", u16[B:2 * B].view(torch.float16).unsqueeze(-1)
                P, d = P.gather(-1, k[..., None]), d.gather(-1, k[..., None])
            else:
                what, half = "probabilities", u16[B:].view(torch.float16).view(B, Cout, *D["Of"]).movedim(1, -1)
                at = half.gather(-1, k[..., None])
                top = half.max(-1, keepdim=True).values
                if not bool((_bits(at.contiguous()) == _bits(top.contiguous())).all()):
                    fails.append("probabilities: at %d position(s) the map's class does not hold the largest "
                                 "probability bit for bit (the top class's value is the confidence 1 / s)"
                                 % int((at != top).sum()))
            bad, excess, st = check_prob(half.to(f64), P, d, A_SM[prec])
            _merge(stats, st)
            if bool(bad.any()):
                fails.append(describe(what, D, bad, excess, half, P, info))
        view(op.out1).copy_(snap.of(op.out1))
    for key, live in restored.items():
        if not torch.equal(_bits(live), _bits(snap.store[key])):
            role = [r for r, t in reach(op) if t.untyped_storage().data_ptr() == key]
            diff = (_bits(live) != _bits(snap.store[key])).nonzero()
            fails.append("moved outside the output window: %d element(s) of the storage behind %s, first at flat "
                         "index %d" % (diff.shape[0], "/".join(role), int(diff[0])))
    return fails, stats


def _whole_of(op, key):
    for _, t in reach(op):
        if t.untyped_storage().data_ptr() == key:
            return _whole(t)
    raise KeyError(key)


def check_classes(got, v, S, lut, c_acc):
    """got: int64 [B, D, H, W] class map; v, S: float64 [B, D, H, W, Cout].  The class is the first index of the
    largest v (through lut when set); another class passes only where its float64 gap to the largest value is within
    the accumulation bound of the two candidates."""
    top, cls = v.max(-1)
    ids = torch.arange(v.shape[-1], device=v.device) if lut is None else torch.tensor(lut, device=v.device)
    mism = got != ids[cls]
    if not bool(mism.any()):
        return None
    vm, Sm = v[mism], S[mism]
    tol = c_acc * (Sm.gather(1, cls[mism][:, None]) + Sm)
    ok = ((ids[None, :] == got[mism][:, None]) & (top[mism][:, None] - vm <= tol)).any(1)
    if bool(ok.all()):
        return None
    at = mism.nonzero()[~ok]
    return ("class map: %d position(s) hold a class whose float64 value is below the largest by more than the "
            "accumulation bound; first (b, d, h, w) = %s: got %d, want %d"
            % (at.shape[0], tuple(at[0].tolist()), int(got[tuple(at[0])]), int(ids[cls[tuple(at[0])]])))


def class_softmax(v):
    """float64 softmax over the last axis: p_c = exp(v_c - max v) / sum_j exp(v_j - max v)"""
    e = torch.exp(v - v.max(-1, keepdim=True).values)
    return e / e.sum(-1, keepdim=True)


def softmax_bound(v, S, c_acc):
    """-> (p, d): the float64 probabilities of the class values v [..., Cout], and d, the bound on how far the error of
    the device's values moves them.  The device's values carry at most delta_j = c_acc S_j each (they are fp32 sums,
    never rounded to the storage type); since dp_c = p_c (dv_c - sum_j p_j dv_j), p_c moves by at most
    p_c (delta_c + sum_j p_j delta_j)."""
    p = class_softmax(v)
    delta = c_acc * S
    return p, p * (delta + (p * delta).sum(-1, keepdim=True))


def chosen_class(got, v, lut):
    """the class index behind each map entry (through lut when set; among classes sharing a label, the largest v), or
    the float64 arg-max where no class has the entry's label"""
    if lut is None:
        ids = torch.arange(v.shape[-1], device=v.device)
    else:
        ids = torch.tensor(lut, device=v.device)
    match = ids == got[..., None]
    k = torch.where(match, v, torch.full_like(v, -float("inf"))).argmax(-1)
    return torch.where(match.any(-1), k, v.argmax(-1))


def check_prob(got, p, d_val, a_sm):
    """float16 probabilities: |got - p| <= 1/2 ulp_f16(p + d) + d, d = d_val + a_sm p (got, p, d_val: float64 of one
    shape, d_val from softmax_bound; a NaN fails).  a_sm p covers expf, the fp32 sum over the classes and the
    division.  -> (bad, excess, stats): stats 'softmax', the largest (|got - p| - 1/2 ulp_f16 - d_val) / p, what a_sm
    has to cover, and 'softmax_raw', the same without d_val"""
    d = d_val + a_sm * p
    err = (got - p).abs()
    bound = 0.5 * ulp_store(p + d, "f16") + d
    bad = ~(err <= bound)
    e = err - 0.5 * ulp_store(torch.maximum(p, got.abs()), "f16")
    stats = {}
    pos = p > 0
    if bool(pos.any()):
        stats["softmax"] = float(((e - d_val)[pos] / p[pos]).max())
        stats["softmax_raw"] = float((e[pos] / p[pos]).max())
    return bad, err - bound, stats


def describe(what, D, bad, excess, got, ref, info):
    """where the failures of one output lie: the worst element and its tile, and the share of failing positions on a
    tile edge, a tensor edge, or where a tap reads a margin plane"""
    n = int(bad.sum())
    worst = torch.where(bad, excess, torch.full_like(excess, -1.0)).flatten().argmax()
    idx = []
    for s in reversed(bad.shape):
        idx.append(int(worst % s))
        worst = worst // s
    b, d, h, w, c = reversed(idx)
    pos = bad.any(-1).any(0).nonzero()                                  # failing (d, h, w) on the full grid
    om, O = D["omul"], D["O"]
    o = torch.stack([pos[:, i] // om[i] for i in range(3)], 1)          # iteration-space coordinates
    msg = ["%s: %d element(s) beyond the bound; worst (b, d, h, w, c) = %s: got %r, float64 %r, %.3g beyond"
           % (what, n, (b, d, h, w, c), float(got[b, d, h, w, c]), float(ref[b, d, h, w, c]),
              float(excess[b, d, h, w, c]))]
    Ot = torch.tensor(O, device=o.device)
    tensor_edge = ((o == 0) | (o == Ot - 1))[:, [i for i in range(3) if O[i] > 1]].any(1)
    share = ["tensor edge %d/%d" % (int(tensor_edge.sum()), pos.shape[0])]
    if info is not None:
        T = [max(1, info[k]) for k in ("TD", "TH", "TW")]
        Tt = torch.tensor(T, device=o.device)
        off = o % Tt
        tile_edge = ((off == 0) | (off == Tt - 1))[:, [i for i in range(3) if T[i] > 1]].any(1)
        share.append("tile edge %d/%d" % (int(tile_edge.sum()), pos.shape[0]))
        wo = (d // om[0], h // om[1], w // om[2])
        msg.append("worst in tile %s at offset %s of box %s"
                   % (tuple(wo[i] // T[i] for i in range(3)), tuple(wo[i] % T[i] for i in range(3)), tuple(T)))
    if D["src_d0"] > 0:
        dz = [t[1] for t in D["taps"]]
        dlen = D["ID"] - 2 * D["src_d0"]
        z = o[:, 0] * D["stride"][0]
        margin = (z + min(dz) < 0) | (z + max(dz) >= dlen)
        share.append("reading a margin plane %d/%d" % (int(margin.sum()), pos.shape[0]))
    return "; ".join(msg) + "; failing positions: " + ", ".join(share)
