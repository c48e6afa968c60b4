"""tests/conv_replay.py without a GPU: its float64 reference against torch's float64 convolutions on ConvOps planned
on CPU tensors (the SIMT flavour of occd_conv_plan_create needs no driver), the sharpness of its comparator on results
corrupted on the host, and the census of distinct launches the six shipped configurations plan."""
import contextlib
import copy
import io
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

import conv_replay as R
from occdepth_b200 import _lib
from occdepth_b200.engine import CL, ConvOp, Plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f64 = torch.float64


@pytest.fixture(autouse=True)
def simt(monkeypatch):
    monkeypatch.setenv("OCCDEPTH_CONV_IMPL", "simt")
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")


def g16(*shape, seed=0, scale=1.0):
    """seeded values every storage type holds exactly"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).float()


def planar(t):
    """channels-last [B, D, H, W, C] -> float64 [B, C, D, H, W]"""
    return t.permute(0, 4, 1, 2, 3).to(f64)


def cl_last(t):
    return t.permute(0, 2, 3, 4, 1)


def close(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    rel = float((a - b).abs().max() / b.abs().max())
    assert rel <= 1e-12, rel


def window(plan, B, D, H, W, C, cstride, coff, halo=0):
    """a channel window of a wider buffer, optionally with margin planes"""
    buf = torch.zeros(B, D + 2 * halo, H, W, cstride, dtype=plan.dtype)
    return CL(buf, C, coff, halo, D)


def prepared(op, seed=1):
    R.fill(op, seed)
    snap = R.Snapshot(op)
    return snap, R.reference(snap)


def src64(snap, i=0):
    D = snap.D
    return planar(snap.srcs[i][..., D["src_coff"][i]:D["src_coff"][i] + D["src_C"][i]])


def fake(op, weight=None, edit=None, **fields):
    """an op with descriptor fields no driverless plan accepts (tap groups, per-image weights): the reference reads
    the descriptor and the tensors only"""
    d = _lib.ConvDesc.from_buffer_copy(op.desc)
    for k, val in fields.items():
        setattr(d, k, val)
    if edit is not None:
        edit(d)
    return types.SimpleNamespace(desc=d, srcs=op.srcs, out0=op.out0, res1=op.res1, res2=op.res2, out1=op.out1,
                                 out1_mode=op.out1_mode, weight=op.weight if weight is None else weight, bias=op.bias,
                                 weight_runtime=False, lut=op.lut, impl=_lib.CONV_IMPL_SIMT)


# ---------------------------------------------------------------------------------------------------------------
# reference against torch
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_dense_stride_dilation_padding_windows_margins(precision):
    """strided / dilated / padded dense convs whose source and output are channel windows of wider buffers; the second
    reads non-zero margin planes"""
    plan = Plan(torch.device("cpu"), precision=precision)
    w, b = g16(20, 24, 3, 3, 3, scale=0.1), g16(20, seed=2)
    x = window(plan, 2, 7, 9, 10, 24, 40, 8)
    out = window(plan, 2, 7, 5, 3, 20, 48, 16)
    plan.conv(x, w, b, stride=(1, 2, 2), padding=(2, 1, 0), dilation=(2, 1, 2), act="leaky", out=out)
    snap, ref = prepared(plan.ops[-1])
    want = F.leaky_relu(F.conv3d(src64(snap), w.to(f64), b.to(f64), (1, 2, 2), (2, 1, 0), (2, 1, 2)), 0.01)
    close(ref.out0[..., :20], cl_last(want))
    assert bool(ref.mask.all()) and float(ref.out0[..., 20:].abs().max()) == 0
    # margins: 2 planes each side, holding data; the conv is 'same' over the 6 interior planes
    x = window(plan, 1, 6, 5, 8, 24, 32, 8, halo=2)
    plan.conv(x, w, b, padding=(2, 1, 1), dilation=(2, 1, 1), act="none", out=window(plan, 1, 6, 5, 8, 20, 24, 0, 2))
    snap, ref = prepared(plan.ops[-1])
    assert snap.D["src_d0"] == 2 and snap.D["ID"] == 10 and float(snap.srcs[0][:, :2].abs().max()) > 0
    want = F.conv3d(src64(snap), w.to(f64), b.to(f64), 1, (2, 1, 1), (2, 1, 1))[:, :, 2:8]
    close(ref.v[..., :20], cl_last(want))
    assert float((ref.S - ref.v.abs()).min()) >= 0


def test_pool_2x2x2():
    """AvgPool3d(2) + 1x1x1 conv as one strided 8-tap conv"""
    plan = Plan(torch.device("cpu"), precision="tf32")
    w1, b = g16(16, 8, 1, 1, 1), g16(16, seed=3)
    plan.conv(plan.alloc(1, 4, 6, 8, 8), (w1 / 8).expand(16, 8, 2, 2, 2).contiguous(), b, stride=2)
    snap, ref = prepared(plan.ops[-1])
    close(ref.out0, cl_last(F.conv3d(F.avg_pool3d(src64(snap), 2), w1.to(f64), b.to(f64))))


def test_transposed_conv_eight_launches_and_grouped():
    plan = Plan(torch.device("cpu"), precision="tf32")
    w, b = g16(16, 8, 3, 3, 3, scale=0.2), g16(8, seed=4)
    x = plan.alloc(1, 3, 4, 5, 16)
    skip = plan.alloc(1, 6, 8, 10, 8)
    plan.conv_transpose_k3s2(x, w, b, act="relu", res_post=skip)
    assert len(plan.ops) == 8
    R.fill(plan.ops[0], 5)                              # all eight share x, skip and y
    snap = R.Snapshot(plan.ops[0])
    want = F.relu(F.conv_transpose3d(src64(snap), w.to(f64), b.to(f64), 2, 1, 1)) + planar(snap.res2[..., :8])
    got = torch.zeros(1, 6, 8, 10, 8, dtype=f64)
    seen = torch.zeros(6, 8, 10, dtype=torch.int32)
    for op in plan.ops:
        ref = R.reference(R.Snapshot(op))
        got[:, ref.mask] = ref.out0[:, ref.mask]
        seen += ref.mask
        assert int(ref.mask.sum()) == 3 * 4 * 5
    assert bool((seen == 1).all())
    close(got, cl_last(want))
    # the same eight phases as tap groups of ONE launch
    ops = sorted(plan.ops, key=lambda o: -o.desc.n_taps)
    taps = [t for o in ops for t in R.desc_fields(o)["taps"]]
    tap0 = [0]
    for o in ops:
        tap0.append(tap0[-1] + o.desc.n_taps)

    def edit(d):
        d.n_taps, d.n_groups = len(taps), 8
        for i, t in enumerate(taps):
            d.taps[i].src, d.taps[i].dz, d.taps[i].dy, d.taps[i].dx = t
        d.group_tap0[:9] = tap0
        for g, o in enumerate(ops):
            d.group_oadd[g][:] = list(o.desc.oadd)
    grouped = fake(ops[0], weight=torch.cat([o.weight for o in ops]), edit=edit)
    ref = R.reference(R.Snapshot(grouped))
    assert bool(ref.mask.all())
    close(ref.out0, cl_last(want))


def test_three_source_sum_with_residual():
    """the ASPP stage: three sources, dilations 1 / 2 / 3, one accumulator, residual before the relu"""
    plan = Plan(torch.device("cpu"), precision="bf16")
    xs = [plan.alloc(1, 6, 7, 8, 16) for _ in range(3)]
    ws = [g16(16, 16, 3, 3, 3, seed=i, scale=0.1) for i in range(3)]
    b = g16(16, seed=9)
    res = window(plan, 1, 6, 7, 8, 16, 32, 16)
    plan.conv_multi(xs, ws, b, [1, 2, 3], [1, 2, 3], act="relu", res1=res)
    snap, ref = prepared(plan.ops[-1])
    acc = sum(F.conv3d(src64(snap, i), w.to(f64), None, 1, d, d) for i, (w, d) in enumerate(zip(ws, (1, 2, 3))))
    want = F.relu(acc + b.to(f64).view(1, -1, 1, 1, 1) + planar(snap.res1[..., 16:32]))
    close(ref.out0, cl_last(want))


def test_per_image_weights():
    plan = Plan(torch.device("cpu"), precision="tf32")
    b = g16(24, seed=1)
    x = plan.alloc(2, 1, 5, 6, 40)
    plan.conv(x, g16(24, 40, 1, 1, 1), b)
    op = plan.ops[-1]
    D = R.desc_fields(op)
    wb = torch.zeros(2, D["Cout_pad"], D["Kpad"])
    wb[:, :24, :40] = g16(2, 24, 40, seed=7)
    snap, ref = prepared(fake(op, weight=wb, weight_per_image=1))
    for i in range(2):
        want = F.conv3d(src64(snap)[i:i + 1], wb[i, :24, :40, None, None, None].to(f64), b.to(f64))
        close(ref.out0[i:i + 1], cl_last(want))


@pytest.mark.parametrize("post", [False, True])
def test_residual_placements_and_channels_last_out1(post):
    """res1 and res2 before the activation, or res2 after it; out1 (channels-last) is the pre-activation value"""
    plan = Plan(torch.device("cpu"), precision="tf32")
    w, b = g16(12, 16, 1, 3, 3, scale=0.2), g16(12, seed=2)
    x = plan.alloc(2, 1, 9, 11, 16)
    r1, r2 = plan.alloc(2, 1, 9, 11, 12), window(plan, 2, 1, 9, 11, 12, 32, 8)
    pre = window(plan, 2, 1, 9, 11, 12, 24, 8)
    plan.conv(x, w, b, padding=(0, 1, 1), act="silu", res1=r1, res2=r2, res2_post=post, out1=pre, out1_mode="cl")
    snap, ref = prepared(plan.ops[-1])
    r1p, r2p = planar(snap.res1[..., :16]), planar(snap.res2[..., 8:24])
    v = F.conv3d(src64(snap), w.to(f64), b.to(f64), 1, (0, 1, 1)) + r1p[:, :12] + (0 if post else r2p[:, :12])
    close(ref.v[..., :12], cl_last(v))
    close(ref.out0[..., :12], cl_last(F.silu(v) + (r2p[:, :12] if post else 0)))
    # pad channels 12..15: what the epilogue makes of a zero accumulator -- it reads the residuals' channels there
    vp = r1p[:, 12:16] + (0 if post else r2p[:, 12:16])
    close(ref.out0[..., 12:], cl_last(F.silu(vp) + (r2p[:, 12:16] if post else 0)))


def test_planar_and_class_map_out1():
    plan = Plan(torch.device("cpu"), precision="tf32")
    w, b = g16(12, 16, 3, 3, 3, scale=0.2), g16(12, seed=2)
    x = plan.alloc(2, 4, 5, 6, 16)
    logits = torch.zeros(2, 17, 4, 5, 6)
    plan.conv(x, w, b, padding=1, act="sigmoid", out1=logits, out1_mode="planar", out1_coff=3)
    snap, ref = prepared(plan.ops[-1])
    v = F.conv3d(src64(snap), w.to(f64), b.to(f64), 1, 1)
    close(ref.v[..., :12], cl_last(v))
    close(ref.out0[..., :12], cl_last(torch.sigmoid(v)))
    assert float((ref.out0[..., 12:] - 0.5).abs().max()) == 0          # sigmoid of the zero pad accumulator
    # class map with a label remap: first index of the largest value, through the lut
    lut = tuple(range(40, 52))
    cm = torch.zeros(2, 4, 5, 6, dtype=torch.uint16)
    plan.conv(x, w, b, padding=1, out1=cm, out1_mode="classes", no_out0=True, lut=lut)
    op = plan.ops[-1]
    if op.out1_mode != "classes":
        pytest.skip("the driverless kernel writes no class map")
    snap, ref = prepared(op)
    v = F.conv3d(src64(snap), w.to(f64), b.to(f64), 1, 1)
    want = v.argmax(1) + 40
    assert R.check_classes(want, ref.v[..., :12], ref.S[..., :12], lut, R.C_ACC["tf32"] * snap.K ** 0.5) is None
    emulate(op, snap, ref)
    assert R.check_op(op, snap, ref)[0] == []
    # a neighbouring class passes only where the two values are within the accumulation bound: not here
    other = torch.where(want > 40, want - 1, want + 1)
    assert "class map" in R.check_classes(other, ref.v[..., :12], ref.S[..., :12], lut, R.C_ACC["tf32"] * snap.K ** 0.5)
    R._bits(op.out1)[0, 0, 0, 0] = int(other[0, 0, 0, 0])
    assert any("class map" in f for f in R.check_op(op, snap, ref)[0])


# ---------------------------------------------------------------------------------------------------------------
# the comparator
def emulate(op, snap, ref, v=None, out0=None, mode=None, probs=None):
    """store into the op's live buffers what a correct device stores (mode: the rounding, default the type's own;
    probs: the class probabilities [..., Cout] to store in place of the float64 softmax of v)"""
    D, prec, Cw, m = snap.D, snap.precision, ref.Cw, ref.mask
    v = ref.v if v is None else v
    if D["out0"]:
        store = "fp32" if (D["out0_exact"] and prec == "tf32") else prec
        q = R.quantize(ref.out0 if out0 is None else out0, store, mode)
        win = op.out0.interior()[..., D["out0_coff"]:D["out0_coff"] + Cw]
        win[:, m] = q[:, m].to(win.dtype)
    if D["out1_mode"] == _lib.OUT1_CL:
        win = op.out1.interior()[..., D["out1_coff"]:D["out1_coff"] + Cw]
        win[:, m] = R.quantize(v, prec, mode)[:, m].to(win.dtype)
    elif D["out1_mode"] == _lib.OUT1_F32_PLANAR:
        win = cl_last(op.out1)[..., D["out1_coff"]:D["out1_coff"] + D["Cout"]]
        win[:, m] = v[..., :D["Cout"]][:, m].float()
    elif D["out1_mode"] in R.CLASS_OUT1:
        B, Cout = D["B"], D["Cout"]
        u16 = op.out1.reshape(-1, *D["Of"])
        k = v[..., :Cout].argmax(-1)
        cls = k if snap.lut is None else torch.tensor(snap.lut)[k]
        R._bits(u16[:B])[:, m] = cls[:, m].to(torch.int16)
        p = R.class_softmax(v[..., :Cout]) if probs is None else probs
        if D["out1_mode"] == _lib.OUT1_CLASS_U16_CONF:
            R._bits(u16[B:2 * B])[:, m] = f16_bits(p.gather(-1, k[..., None])[..., 0], mode)[:, m]
        elif D["out1_mode"] == _lib.OUT1_CLASS_U16_PROBS:
            R._bits(u16[B:]).view(B, Cout, *D["Of"])[:] = f16_bits(p, mode).movedim(-1, 1)


def f16_bits(p, mode=None):
    """float16 bits of p (float64 >= 0): nearest even, or toward zero for mode 'trunc'"""
    h = p.to(torch.float16)
    bits = R._bits(h).clone()
    if mode == "trunc":
        bits -= (h.to(f64) > p).to(torch.int16)
    return bits


def _case(precision, out1=True):
    """3x3x3 conv, 20 of 24 stored channels real, residual + relu, out0 a window of a wider buffer, planar out1"""
    plan = Plan(torch.device("cpu"), precision=precision)
    w, b = g16(20, 32, 3, 3, 3, scale=0.05), g16(20, seed=2)
    x = plan.alloc(1, 5, 6, 8, 32)
    res = plan.alloc(1, 5, 6, 8, 24)
    out = window(plan, 1, 5, 6, 8, 20, 48, 16)
    logits = torch.zeros(1, 23, 5, 6, 8)
    plan.conv(x, w, b, padding=1, act="relu", res1=res, out=out, out1=logits if out1 else None,
              out1_mode="planar" if out1 else "none", out1_coff=2)
    op = plan.ops[-1]
    snap, ref = prepared(op, seed=11)
    return op, snap, ref, w, b


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_comparator_accepts_the_rounded_result_and_an_fp32_reordering(precision):
    op, snap, ref, w, b = _case(precision)
    emulate(op, snap, ref)
    fails, stats = R.check_op(op, snap, ref)
    assert fails == [] and stats["acc"] <= 0
    # the same sum in fp32, in the order of torch's CPU kernel
    v32 = F.conv3d(src64(snap).float(), w, b, 1, 1) + planar(snap.res1[..., :20]).float()
    v = ref.v.clone()
    v[..., :20] = cl_last(v32).to(f64)
    emulate(op, snap, ref, v=v, out0=torch.relu(v))
    fails, stats = R.check_op(op, snap, ref)
    assert fails == [], fails
    assert 0 < stats["acc"] < R.C_ACC[precision]


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_comparator_rejects_truncation_and_one_ulp(precision):
    op, snap, ref, _, _ = _case(precision, out1=False)
    emulate(op, snap, ref, mode="trunc")
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and fails[0].startswith("out0:"), fails
    emulate(op, snap, ref)
    assert R.check_op(op, snap, ref)[0] == []
    # one storage ulp on one element (away from the float64 value)
    win = op.out0.interior()[..., 16:40]
    q = win.to(f64)
    at = tuple(((q > ref.out0) & (ref.out0 > 0.5)).nonzero()[0].tolist())
    win[at] = (q[at] + R.ulp_store(q[at], precision)).to(win.dtype)
    assert float(win[at]) != float(q[at])
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and "1 element(s) beyond the bound" in fails[0] and str(at) in fails[0], fails


def _partial(snap, taps, drop_bias=True):
    """the reference of the same launch with only `taps` (indices) contributing, without bias and residual"""
    s = copy.copy(snap)
    s.weight = snap.weight.clone()
    keep = torch.zeros(s.weight.shape[0], dtype=torch.bool)
    keep[list(taps)] = True
    s.weight[~keep] = 0
    s.bias = torch.zeros_like(snap.bias)
    s.res1 = s.res2 = None
    return R.reference(s).v


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_comparator_rejects_a_dropped_tap_and_a_swapped_neighbour_mask(precision):
    op, snap, ref, _, _ = _case(precision, out1=False)
    taps = snap.D["taps"]
    # one tap missing on one boundary row only: tap (0, +1, 0) at h = 0
    t = taps.index((0, 0, 1, 0))
    v = ref.v.clone()
    v[:, :, 0] -= _partial(snap, [t])[:, :, 0]
    emulate(op, snap, ref, out0=torch.relu(v))
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and "tensor edge" in fails[0], fails
    bad_rows = {int(h) for h in (op.out0.interior()[..., 16:40].to(f64) != R.quantize(ref.out0, precision))
                .nonzero()[:, 2]}
    assert bad_rows == {0}
    # x-packed sum with the W-neighbour masks swapped at w = 0: the dx = +1 partial is masked off and the dx = -1
    # partial of the wrapped lane (last column of the row above) is taken instead
    plus = _partial(snap, [i for i, tp in enumerate(taps) if tp[3] == 1])
    minus = _partial(snap, [i for i, tp in enumerate(taps) if tp[3] == -1])
    v = ref.v.clone()
    v[:, :, :, 0] += -plus[:, :, :, 0] + torch.roll(minus, 1, 2)[:, :, :, -1]
    emulate(op, snap, ref, out0=torch.relu(v))
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and "beyond the bound" in fails[0], fails


def test_comparator_rejects_stray_writes_and_dirty_pad_channels():
    op, snap, ref, _, _ = _case("tf32")
    emulate(op, snap, ref)
    assert R.check_op(op, snap, ref)[0] == []
    buf = op.out0.buf
    for at in [(0, 2, 3, 4, 15), (0, 2, 3, 4, 40)]:             # the channels on either side of the window [16, 40)
        old = float(buf[at])
        buf[at] = old + 1.0
        fails, _ = R.check_op(op, snap, ref)
        assert len(fails) == 1 and "moved outside the output window" in fails[0], fails
        buf[at] = old
    old = float(op.out1[0, 1, 2, 3, 4])                         # planar out1: channel 1 lies before out1_coff = 2
    op.out1[0, 1, 2, 3, 4] = 7.0
    assert any("out1_planar" in f for f in R.check_op(op, snap, ref)[0])
    op.out1[0, 1, 2, 3, 4] = old
    op.srcs[0].buf[0, 0, 0, 0, 0] += 1.0                        # a source
    assert any("src" in f for f in R.check_op(op, snap, ref)[0])
    op.srcs[0].buf[0, 0, 0, 0, 0] -= 1.0
    assert R.check_op(op, snap, ref)[0] == []
    # pad channel 20 of the window: no activation path makes 2^-9 of relu(0 + 0 + res)
    at = (0, 1, 1, 1, 16 + 20)
    buf[at] = float(buf[at]) + 2.0 ** -9
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and "(0, 1, 1, 1, 20)" in fails[0], fails


# ---------------------------------------------------------------------------------------------------------------
# class confidence (mode 4) and class probabilities (mode 5)
CLS_B, CLS_C, CLS_DIMS = 2, 12, (4, 5, 6)
CLS_P = CLS_DIMS[0] * CLS_DIMS[1] * CLS_DIMS[2]


def _class_case(mode, precision="tf32", lut=None):
    """3x3x3 conv of 2 items onto 12 classes writing the map and its confidence (mode 'classes_conf') or every
    probability ('classes_probs'); out1 is the front of a uint16 storage one element longer, so that a store past
    its (rows * B * positions) region lands in the storage"""
    plan = Plan(torch.device("cpu"), precision=precision)
    w, b = g16(CLS_C, 16, 3, 3, 3, scale=0.3), g16(CLS_C, seed=2)
    x = plan.alloc(CLS_B, *CLS_DIMS, 16)
    rows = (2 if mode == "classes_conf" else 1 + CLS_C) * CLS_B
    store = torch.zeros(rows * CLS_P + 1, dtype=torch.uint16)
    shape = (2, CLS_B) if mode == "classes_conf" else (rows,)
    plan.conv(x, w, b, padding=1, out1=store[:rows * CLS_P].view(*shape, *CLS_DIMS), out1_mode=mode, no_out0=True,
              lut=lut)
    op = plan.ops[-1]
    assert op.out1_mode == mode, "the driverless kernel writes no class map"
    snap, ref = prepared(op, seed=5)
    return op, snap, ref, w, b, store


def test_class_softmax_reference_against_torch():
    op, snap, ref, w, b, _ = _class_case("classes_probs")
    v = F.conv3d(src64(snap), w.to(f64), b.to(f64), 1, 1)
    close(ref.v[..., :CLS_C], cl_last(v))
    close(R.class_softmax(ref.v[..., :CLS_C]), cl_last(torch.softmax(v, 1)))
    g = torch.Generator().manual_seed(3)
    u = torch.randn(7, 33, generator=g, dtype=f64) * 30           # wide spreads: probabilities far below 2^-24
    close(R.class_softmax(u), torch.softmax(u, -1))
    p, d = R.softmax_bound(ref.v[..., :CLS_C], ref.S[..., :CLS_C], 1e-6)
    assert float((p.sum(-1) - 1).abs().max()) < 1e-12 and bool((d > 0).all())


@pytest.mark.parametrize("lut", [None, tuple(range(40, 40 + CLS_C))])
@pytest.mark.parametrize("mode", ["classes_conf", "classes_probs"])
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_comparator_class_probs_accepts_the_rounded_result_and_an_fp32_softmax(precision, mode, lut):
    op, snap, ref, _, _, _ = _class_case(mode, precision, lut)
    emulate(op, snap, ref)
    fails, stats = R.check_op(op, snap, ref)
    assert fails == [], fails
    assert stats["softmax_raw"] <= 0 and stats["softmax"] <= 0, stats
    # fp32 values and an fp32 softmax that sums the classes in the opposite order
    v32 = ref.v[..., :CLS_C].float()
    e = torch.exp(v32 - v32.max(-1, keepdim=True).values)
    s = torch.zeros_like(e[..., 0])
    for c in reversed(range(CLS_C)):
        s = s + e[..., c]
    emulate(op, snap, ref, probs=(e / s[..., None]).to(f64))
    fails, stats = R.check_op(op, snap, ref)
    assert fails == [], fails
    assert stats["softmax"] <= R.A_SM[precision], stats


@pytest.mark.parametrize("mode", ["classes_conf", "classes_probs"])
def test_comparator_class_probs_rejects_one_ulp_and_truncation(mode):
    what = "confidence" if mode == "classes_conf" else "probabilities"
    op, snap, ref, _, _, _ = _class_case(mode)
    emulate(op, snap, ref, mode="trunc")
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and fails[0].startswith(what + ":"), fails
    emulate(op, snap, ref)
    assert R.check_op(op, snap, ref)[0] == []
    # one float16 ulp on one stored value above 0.1 that is not the largest of its position
    u16 = op.out1.reshape(-1, *CLS_DIMS)[CLS_B:]
    half = u16.view(torch.float16)
    top = half.view(CLS_B, -1, *CLS_DIMS).max(1, keepdim=True).values.expand(-1, u16.shape[0] // CLS_B, -1, -1, -1)
    cand = (half.view(CLS_B, -1, *CLS_DIMS) > 0.1) & ((half.view(CLS_B, -1, *CLS_DIMS) < top) | (mode == "classes_conf"))
    at = tuple(cand.nonzero()[0].tolist())
    R._bits(u16).view(CLS_B, -1, *CLS_DIMS)[at] += 1
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and fails[0].startswith(what + ": 1 element(s) beyond the bound"), fails


def test_comparator_class_probs_rejects_the_wrong_item_stride():
    """item 1's probabilities stored at out1[B P + pos + n P] (no b (Cout - 1) P): over item 0's rows, one row down"""
    op, snap, ref, _, _, _ = _class_case("classes_probs")
    emulate(op, snap, ref)
    p = R.class_softmax(ref.v[..., :CLS_C])
    rows = op.out1.reshape(-1, CLS_P)
    b = 1
    for n in range(CLS_C):
        R._bits(rows)[CLS_B + b + n] = f16_bits(p[b, ..., n]).reshape(-1)
    fails, _ = R.check_op(op, snap, ref)
    assert any(f.startswith("probabilities:") for f in fails), fails


def test_comparator_class_conf_rejects_swapped_halves():
    op, snap, ref, _, _, _ = _class_case("classes_conf")
    emulate(op, snap, ref)
    u16 = op.out1
    u16.copy_(torch.stack([u16[1].clone(), u16[0].clone()]))          # [2, B, D, H, W]: map, then confidence
    fails, _ = R.check_op(op, snap, ref)
    assert any(f.startswith("class map:") for f in fails) and any(f.startswith("confidence:") for f in fails), fails


@pytest.mark.parametrize("mode", ["classes_conf", "classes_probs"])
def test_comparator_class_probs_rejects_a_store_past_the_region(mode):
    op, snap, ref, _, _, store = _class_case(mode)
    emulate(op, snap, ref)
    assert R.check_op(op, snap, ref)[0] == []
    assert op.out1.numel() == store.numel() - 1
    R._bits(store)[-1] = 0x3C00                          # 1.0 in float16, one element past the map and probabilities
    fails, _ = R.check_op(op, snap, ref)
    assert len(fails) == 1 and "moved outside the output window" in fails[0], fails


def test_signature_tells_launches_apart():
    plan = Plan(torch.device("cpu"), precision="tf32")
    w, b = g16(16, 16, 1, 3, 3), g16(16)
    a = plan.alloc(1, 1, 9, 11, 16)
    for _ in range(2):
        plan.conv(a, w + 1, b, padding=(0, 1, 1))
    plan.conv(window(plan, 1, 1, 9, 11, 16, 32, 8), w, b, padding=(0, 1, 1))
    plan.conv(a, w, b, padding=(0, 1, 1), act="relu")
    plan.conv(a, w, b, padding=(0, 2, 2), dilation=(1, 2, 2))
    sigs = [R.signature(op) for op in plan.ops]
    assert sigs[0] == sigs[1] and len(set(sigs)) == 4
    assert all(dict(s)["kernel"] is None for s in sigs)


# ---------------------------------------------------------------------------------------------------------------
def test_census_of_the_shipped_configurations(capsys):
    """distinct launches per shipped configuration (forward + class-map plans, real shapes): the size of the sweep
    tests/test_gpu_conv_replay.py replays.  Without a driver the kernel-choice fields are absent, so these counts are a
    lower bound of the GPU's."""
    tools = os.path.join(ROOT, "tools")
    if tools not in sys.path:
        sys.path.insert(0, tools)
    import shipped_configs as sc
    import slab_sim
    seen_all = set()
    lines = []
    for name in sc.CONFIGS:
        m, batch, _ = sc.make_case(name)
        B, V, H, W, N, P, dev = slab_sim._shape_args(m, batch)
        sigs, n_ops = set(), 0
        for classes in (None, ("classes", None)):
            with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
                plan = m._build(B, V, H, W, N, P, dev, batch, classes=classes)[0]
            ops = [op for op in plan.ops if isinstance(op, ConvOp)]
            n_ops += len(ops)
            sigs |= {R.signature(op) for op in ops}
            del plan, ops
        lines.append("%-40s %4d conv launches, %4d distinct, %4d not seen in an earlier configuration"
                     % (name, n_ops, len(sigs), len(sigs - seen_all)))
        assert 30 < len(sigs) < n_ops
        seen_all |= sigs
        del m, batch
    with capsys.disabled():
        print("\nconv-replay census (tf32, forward + class-map plans):\n" + "\n".join(lines)
              + "\ntotal distinct over the six configurations: %d" % len(seen_all))
    assert len(seen_all) > 200
