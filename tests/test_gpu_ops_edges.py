"""Kernel-level parity of the layout, EfficientNet, frustum and per-image-weight paths at their edges: channel
windows and pad channels, batch > 1, extents that are not multiples of the block or tile, every tiled depthwise
instantiation, degenerate resize extents, cameras that see part of the grid from behind.  Each reference is plain
torch in float64 on the CPU, run on inputs already rounded to the storage type."""
import math

import pytest
import torch
import torch.nn.functional as F

import gpu_cases as G
import launch_replay as LR

pytestmark = pytest.mark.gpu

PREC = pytest.mark.parametrize("precision", G.PRECISIONS)
TDT = {"tf32": torch.float32, "bf16": torch.bfloat16}
SENTINEL = -448.0          # exact in bf16 and TF32: channels a kernel must not touch keep it

# bounds: twice the largest figure measured on an H100 (OCCDEPTH_PARITY_DIR), never looser than the one-store bound
# G.TOL for outputs rounded to the activation type
STORE_TOL = {                                 # rounded outputs, relative to max |ref|
    "dwconv": {"tf32": 7.5e-4, "bf16": G.TOL["bf16"]},
    "upsample": {"tf32": 6.5e-4, "bf16": G.TOL["bf16"]},
    "se_fold": {"tf32": 5.3e-4, "bf16": G.TOL["bf16"]},
    "conv_per_image": {"tf32": 7.5e-4, "bf16": G.TOL["bf16"]},
}
SE_GATE_TOL = 5e-7         # sigmoid gates (fast-math exp), absolute
SE_HIDDEN_TOL = 2e-7       # SiLU hidden units, relative to max |ref|
POOL_TOL = 9.5e-8          # squeeze sums, relative to max |sum|
# sampled prior, relative to max |ref|: the sampling coordinates differ from the reference's in fp32 operation order
FRUSTUM_TOL = {"fp32": 6e-6, "f64": 1.6e-5}
GRID_PRIOR_TOL = {"fp32": 2.8e-6, "f64": 6.3e-6}     # given grids: fp32 interpolation only


def L():
    from occdepth_b200 import _lib
    return _lib.lib()


def st():
    from occdepth_b200 import _lib
    return _lib.stream_ptr()


def code(precision):
    return 0 if precision == "tf32" else 1


# ---- planar <-> channels-last ---------------------------------------------------------------------------------------
@PREC
def test_planar_cl_roundtrip(precision):
    """B = 3, S and C not multiples of 32, cstride > C: pad channels zero, values rounded to the activation type
    (TF32 for F32 activations, like every other F32 activation store), and the way back is exact"""
    g = torch.Generator().manual_seed(11)
    B, C_, S, cs = 3, 45, 999, 56
    x = torch.randn(B, C_, S, generator=g) * torch.logspace(-3, 3, C_).view(1, C_, 1)
    xd = x.cuda()
    out = torch.full((B, S, cs), SENTINEL, dtype=TDT[precision], device="cuda")
    assert L().occd_planar_to_cl(xd.data_ptr(), out.data_ptr(), code(precision), B, C_, S, cs, st()) == 0
    got = out.cpu()
    want = x.permute(0, 2, 1)
    if precision == "bf16":
        assert torch.equal(got[..., :C_], want.to(torch.bfloat16))
    else:
        assert torch.equal(got[..., :C_], G.tf32r(want))
    assert torch.all(got[..., C_:] == 0)
    back = torch.full((B * C_ * S + 64,), SENTINEL, device="cuda")
    assert L().occd_cl_to_planar(out.data_ptr(), code(precision), back.data_ptr(), B, C_, S, cs, st()) == 0
    back = back.cpu()
    assert torch.equal(back[:B * C_ * S].view(B, C_, S), got[..., :C_].float().permute(0, 2, 1))
    assert torch.all(back[B * C_ * S:] == SENTINEL)
    # values already of the activation type pass through unchanged
    xr = G.rnd(precision)(x)
    out2 = torch.empty(B, S, cs, dtype=TDT[precision], device="cuda")
    assert L().occd_planar_to_cl(xr.cuda().data_ptr(), out2.data_ptr(), code(precision), B, C_, S, cs, st()) == 0
    back2 = torch.empty(B, C_, S, device="cuda")
    assert L().occd_cl_to_planar(out2.data_ptr(), code(precision), back2.data_ptr(), B, C_, S, cs, st()) == 0
    assert torch.equal(back2.cpu(), xr)


@PREC
def test_copy_channels_and_transpose_windows(precision):
    g = torch.Generator().manual_seed(12)
    tdt, c = TDT[precision], code(precision)
    pos = 333
    src = G.rnd(precision)(torch.randn(pos, 40, generator=g)).to(tdt)
    dst = torch.full((pos, 56), SENTINEL, dtype=tdt, device="cuda")
    assert L().occd_copy_channels(src.cuda().data_ptr(), dst.data_ptr(), c, pos, 24, 40, 8, 56, 24, st()) == 0
    d = dst.cpu()
    assert torch.equal(d[:, 24:48], src[:, 8:32])
    assert torch.all(d[:, :24] == SENTINEL) and torch.all(d[:, 48:] == SENTINEL)
    B, P, C_, cs, coff, ldo = 2, 45, 20, 40, 8, 64
    bstride = 32 * ldo + 128                              # larger than dense
    a = G.rnd(precision)(torch.randn(B, P, cs, generator=g)).to(tdt)
    wt = torch.full((B * bstride,), SENTINEL, dtype=tdt, device="cuda")
    assert L().occd_cl_transpose(a.cuda().data_ptr(), wt.data_ptr(), c, B, P, C_, cs, coff, ldo, bstride, st()) == 0
    w = wt.cpu()
    expect = torch.full((B * bstride,), SENTINEL, dtype=tdt)
    for b in range(B):
        blk = expect[b * bstride:b * bstride + C_ * ldo].view(C_, ldo)
        blk[:, :P] = a[b, :, coff:coff + C_].t()
    assert torch.equal(w, expect)


# ---- squeeze-excite -------------------------------------------------------------------------------------------------
def _se_params(g, B, C_, R, hw):
    pool = (torch.randn(B, C_, generator=g) * 0.5 * hw * 2 ** 24).round().to(torch.int64)
    w1, b1 = torch.randn(R, C_, generator=g) / C_ ** 0.5, torch.randn(R, generator=g)
    w2, b2 = torch.randn(C_, R, generator=g) / R ** 0.5, torch.randn(C_, generator=g)
    mean = pool.double() / 2 ** 24 / hw
    hidden = F.silu(mean @ w1.double().t() + b1.double())
    gate = torch.sigmoid(hidden @ w2.double().t() + b2.double())
    return pool, w1, b1, w2, b2, hidden, gate


def test_se_gate():
    """B = 2, C = 640 (three blocks of the expand FC), R = 160: gates, the hidden layer staged behind them, and the
    squeeze sums cleared for the next forward"""
    g = torch.Generator().manual_seed(13)
    B, C_, R, hw = 2, 640, 160, 53.0
    pool, w1, b1, w2, b2, hidden, gate = _se_params(g, B, C_, R, hw)
    d = lambda t: t.contiguous().cuda()
    bufs = [d(pool), d(w1), d(b1), d(w2.t()), d(b2)]
    out = torch.full((B * C_ + B * R + 16,), SENTINEL, device="cuda")
    assert L().occd_se_gate_fwd(bufs[0].data_ptr(), 1.0 / hw, bufs[1].data_ptr(), bufs[2].data_ptr(),
                                bufs[3].data_ptr(), bufs[4].data_ptr(), out.data_ptr(), B, C_, R, st()) == 0
    o = out.cpu().double()
    eg = float((o[:B * C_].view(B, C_) - gate).abs().max())
    eh = float((o[B * C_:B * C_ + B * R].view(B, R) - hidden).abs().max() / hidden.abs().max())
    G.record("se_gate", "fp32", gate_abs=eg, hidden_rel=eh)
    assert eg <= SE_GATE_TOL and eh <= SE_HIDDEN_TOL
    assert torch.all(o[B * C_ + B * R:] == SENTINEL)
    assert int(bufs[0].abs().max()) == 0


@PREC
def test_scale_weights_pad_columns(precision):
    """C < Kpad, Kpad not a multiple of 256: one rounding of one fp32 product per weight, pad columns exactly 0"""
    g = torch.Generator().manual_seed(14)
    rows, Kpad, C_ = 40, 200, 180
    master = torch.randn(rows, Kpad, generator=g)
    gate = torch.rand(C_, generator=g)
    out = torch.full((rows, Kpad), SENTINEL, dtype=TDT[precision], device="cuda")
    assert L().occd_scale_weights(master.cuda().data_ptr(), gate.cuda().data_ptr(), out.data_ptr(), code(precision),
                                  rows, Kpad, C_, st()) == 0
    got = out.cpu()
    want = G.rnd(precision)(master[:, :C_] * gate).to(TDT[precision])
    assert torch.equal(got[:, :C_], want)
    assert torch.all(got[:, C_:] == 0)


@PREC
def test_se_gate_fold_per_image(precision):
    """B = 2 images with different squeeze sums, Kpad = 328 / C = 320 (two K blocks and padded columns), rows that
    split into several row blocks: one folded weight set per image"""
    g = torch.Generator().manual_seed(15)
    B, C_, R, rows, Kpad, hw = 2, 320, 80, 200, 328, 41.0
    pool, w1, b1, w2, b2, hidden, gate = _se_params(g, B, C_, R, hw)
    master = torch.randn(rows, Kpad, generator=g)
    d = lambda t: t.contiguous().cuda()
    bufs = [d(pool), d(w1), d(b1), d(w2.t()), d(b2), d(master)]
    hid = torch.zeros(B, R, device="cuda")
    out = torch.full((B, rows, Kpad), SENTINEL, dtype=TDT[precision], device="cuda")
    assert L().occd_se_gate_fold_fwd(bufs[0].data_ptr(), 1.0 / hw, bufs[1].data_ptr(), bufs[2].data_ptr(),
                                     bufs[3].data_ptr(), bufs[4].data_ptr(), hid.data_ptr(), bufs[5].data_ptr(),
                                     out.data_ptr(), code(precision), B, C_, R, rows, Kpad, st()) == 0
    got = out.float().cpu()
    assert torch.all(got[:, :, C_:] == 0)
    # each image against its own gates (they differ: a shared weight set would fail)
    assert float((gate[0] - gate[1]).abs().max()) > 0.1
    err = max(G.rel_err(got[b, :, :C_].double(), master[:, :C_].double() * gate[b]) for b in range(B))
    eh = float((hid.cpu().double() - hidden).abs().max() / hidden.abs().max())
    G.record("se_gate_fold", precision, rel=err, hidden_rel=eh)
    assert err <= STORE_TOL["se_fold"][precision], err
    assert eh <= SE_HIDDEN_TOL
    assert int(bufs[0].abs().max()) == 0


# ---- depthwise conv ------------------------------------------------------------------------------------------------
def dw_choice(B, OH, OW, C_, S, n_sms, precision):
    """(cvb, TH, PX) of the tiled kernel: dwt::choose (csrc/dwconv_tiled.cuh) and launch_dw_tiled_ks (OCCD_DW_PX
    unset)"""
    f32 = precision == "tf32"
    cvb = 4 if (C_ < 64 or f32) else 8
    if cvb == 4:
        th = 16
    elif S == 2:
        th = 8
    else:
        th = 16 if B * -(-OH // 16) * -(-OW // 16) * -(-C_ // 64) >= 4 * n_sms else 8
    px = 8 if (cvb == 4 and f32 and S == 1) else 4
    return cvb, th, px


DW_CASES = {
    # id: (precision, B, C, H, W, K, stride, act, cs_in, cs_out)
    "f32_s1_k3_none": ("tf32", 3, 40, 23, 37, 3, 1, "none", 48, 56),
    "f32_s2_k5_relu": ("tf32", 3, 24, 31, 45, 5, 2, "relu", 32, 40),
    "f32_s1_k3_leaky": ("tf32", 3, 72, 19, 26, 3, 1, "leaky", 80, 88),
    "f32_s2_k5_sigmoid": ("tf32", 3, 136, 17, 33, 5, 2, "sigmoid", 144, 136),
    "bf16_c56_s1_k5_leaky": ("bf16", 3, 56, 21, 35, 5, 1, "leaky", 64, 72),
    "bf16_c72_s2_k3_sigmoid": ("bf16", 3, 72, 40, 50, 3, 2, "sigmoid", 80, 88),
    "bf16_c136_s1_k5_relu": ("bf16", 3, 136, 24, 40, 5, 1, "relu", 136, 152),
    "bf16_c200_s1_k3_none_tall": ("bf16", 3, 200, 128, 128, 3, 1, "none", 208, 216),
}
ACTS = {"none": (0, lambda t: t), "relu": (1, F.relu), "leaky": (2, lambda t: F.leaky_relu(t, 0.01)),
        "sigmoid": (4, torch.sigmoid)}


def test_dw_cases_cover_every_tiled_instantiation():
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    reached = set()
    for prec, B, C_, H, W, K, S, *_ in DW_CASES.values():
        reached.add((prec,) + dw_choice(B, math.ceil(H / S), math.ceil(W / S), C_, S, n_sms, prec))
    assert reached == {("tf32", 4, 16, 8), ("tf32", 4, 16, 4), ("bf16", 4, 16, 4), ("bf16", 8, 8, 4),
                       ("bf16", 8, 16, 4)}


@pytest.mark.parametrize("variant", ["tiled", "direct"])
@pytest.mark.parametrize("case", sorted(DW_CASES))
def test_dwconv_windows_acts_batches(case, variant):
    """channel strides wider than C (the input's pad channels hold NaN, the output's must keep their sentinel), every
    activation but SiLU (test_gpu_ops covers it), three images with their own squeeze sums"""
    precision, B, C_, H, W, K, S, act, cs_in, cs_out = DW_CASES[case]
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    tdt = TDT[precision]
    x = G.rnd(precision)(torch.randn(B, C_, H, W, generator=g))
    w = torch.randn(C_, 1, K, K, generator=g) / K
    bias = torch.randn(C_, generator=g)
    OH, OW = math.ceil(H / S), math.ceil(W / S)
    ph, pw = max((OH - 1) * S + K - H, 0), max((OW - 1) * S + K - W, 0)
    ref = F.conv2d(F.pad(x.double(), [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]), w.double(), bias.double(), S, 0,
                   1, C_)
    ref = ACTS[act][1](ref)
    xin = torch.full((B, H, W, cs_in), float("nan"), dtype=tdt)
    xin[..., :C_] = x.permute(0, 2, 3, 1).to(tdt)
    xin = xin.cuda()
    y = torch.full((B, OH, OW, cs_out), SENTINEL, dtype=tdt, device="cuda")
    wk = w.reshape(C_, K * K).t().contiguous().cuda()
    pool = torch.zeros(B, C_, dtype=torch.int64, device="cuda")
    fn = L().occd_dwconv2d_tiled_fwd if variant == "tiled" else L().occd_dwconv2d_fwd
    assert fn(xin.data_ptr(), wk.data_ptr(), bias.cuda().data_ptr(), y.data_ptr(), pool.data_ptr(), code(precision),
              B, H, W, OH, OW, C_, cs_in, cs_out, K, S, ph // 2, pw // 2, ACTS[act][0], st()) == 0
    yc = y.float().cpu()
    assert torch.all(yc[..., C_:] == SENTINEL)
    got = yc[..., :C_].permute(0, 3, 1, 2)
    err = G.rel_err(got.double(), ref)
    if precision == "tf32":
        assert torch.equal(got, G.tf32r(got))
    sums = pool.cpu().double() / 2 ** 24
    want_sums = got.double().sum((2, 3))                 # squeeze of what the next layer reads (the stored values)
    es = float((sums - want_sums).abs().max() / want_sums.abs().max())
    G.record("dwconv_edges.%s.%s" % (case, variant), precision, rel=err, pool_rel=es)
    assert err <= STORE_TOL["dwconv"][precision], err
    assert es <= POOL_TOL, es


# ---- bilinear resize, align_corners=True ----------------------------------------------------------------------------
@PREC
@pytest.mark.parametrize("h,w,OH,OW", [(7, 9, 12, 22), (5, 6, 1, 1), (1, 9, 4, 17), (6, 1, 11, 3), (9, 13, 1, 20)])
def test_upsample_windows_and_degenerate_extents(precision, h, w, OH, OW):
    g = torch.Generator().manual_seed(h * 100 + OW)
    tdt = TDT[precision]
    B, C_, cs_in, in_off, cs_out, out_off = 2, 24, 48, 16, 56, 8
    x = G.rnd(precision)(torch.randn(B, C_, h, w, generator=g))
    ref = F.interpolate(x.double(), size=(OH, OW), mode="bilinear", align_corners=True)
    xin = torch.full((B, h, w, cs_in), float("nan"), dtype=tdt)
    xin[..., in_off:in_off + C_] = x.permute(0, 2, 3, 1).to(tdt)
    y = torch.full((B, OH, OW, cs_out), SENTINEL, dtype=tdt, device="cuda")
    assert L().occd_upsample_bilinear_ac(xin.cuda().data_ptr(), y.data_ptr(), code(precision), B, h, w, OH, OW, C_,
                                         cs_in, in_off, cs_out, out_off, st()) == 0
    yc = y.float().cpu()
    assert torch.all(yc[..., :out_off] == SENTINEL) and torch.all(yc[..., out_off + C_:] == SENTINEL)
    got = yc[..., out_off:out_off + C_].permute(0, 3, 1, 2)
    err = G.rel_err(got.double(), ref)
    G.record("upsample_edges.%dx%d_%dx%d" % (h, w, OH, OW), precision, rel=err)
    assert err <= STORE_TOL["upsample"][precision], err


# ---- frustum sampler ------------------------------------------------------------------------------------------------
IMG_HW = (96, 320)
DMIN, DMAX, DN = 2.0, 58.0, 16
GRID = (23, 20, 7)                                     # 3220 voxels: not a multiple of the 256-thread block
PC_MIN, PC_MAX = (0.0, -25.6, -2.0), (51.2, 25.6, 4.4)


def _cameras(V):
    """KITTI-like lidar->camera transforms (x forward -> camera z).  The cameras sit 10 m into the grid, so the voxels
    behind them and those closer than dmin take the NaN-bin (-2) path; view 1 is a stereo partner, view 2 is turned
    by 0.2 rad.  ida scales by 0.9 and crops, as the dataset augmentation builds it."""
    cams = []
    for v in range(V):
        T = torch.tensor([[0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 1.2], [1.0, 0.0, 0.0, -10.0], [0.0, 0.0, 0.0, 1.0]])
        if v == 1:
            T[0, 3] = -0.54
        if v == 2:
            c, s = math.cos(0.2), math.sin(0.2)
            T = torch.tensor([[c, 0.0, -s, 0.0], [0.0, 1.0, 0.0, 0.0], [s, 0.0, c, 0.0], [0.0, 0.0, 0.0, 1.0]]) @ T
        K4 = torch.tensor([[120.0, 0.0, 160.0, 0.0], [0.0, 120.0, 48.0, 0.0], [0.0, 0.0, 1.0, 0.0],
                           [0.0, 0.0, 0.0, 1.0]])
        ida = torch.tensor([[0.9, 0.0, 0.0, -8.0], [0.0, 0.9, 0.0, -4.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])
        cams.append((T, K4, ida))
    return cams


def _frustum_grid_f64(T, K4, ida):
    return LR.frustum_grid_f64(T.double() @ _grid_to_lidar().double(), K4, ida, GRID, IMG_HW, DN, DMIN, DMAX)


_sample_mean = LR.sample_mean


def _to_kernel_order(r, perm_xzy):
    X, Y, Z = GRID
    return r.view(X, Y, Z).permute(0, 2, 1).reshape(-1) if perm_xzy else r


@pytest.mark.parametrize("V", [1, 2, 3])
@pytest.mark.parametrize("mean_mode,perm_xzy", [(1, 0), (0, 1), (1, 1), (0, 0)])
def test_frustum_sample(V, mean_mode, perm_xzy):
    from oracle import functional as OF
    g = torch.Generator().manual_seed(V)
    h, w = 12, 40
    depth = torch.randn(V, DN, h, w, generator=g).softmax(1)
    cams = _cameras(V)
    table = torch.stack([torch.cat([(T @ _grid_to_lidar())[:3].reshape(-1), K4[:3].reshape(-1), ida.reshape(-1)])
                         for T, K4, ida in cams])
    out = torch.full((GRID[0] * GRID[1] * GRID[2],), float("nan"), device="cuda")
    assert L().occd_frustum_sample_fwd(depth.cuda().data_ptr(), table.cuda().data_ptr(), V, DN, h, w, *GRID,
                                       float(IMG_HW[1]), float(IMG_HW[0]), DMIN, DMAX, mean_mode, out.data_ptr(),
                                       perm_xzy, st()) == 0
    got = out.cpu().double()
    g32 = [OF.frustum_grid(list(GRID), torch.tensor(PC_MIN), torch.tensor(PC_MAX), T, K4, ida, IMG_HW, DN, DMIN, DMAX)
           for T, K4, ida in cams]
    r32, m32 = _sample_mean(depth, g32, mean_mode)
    r64, m64 = _sample_mean(depth.double(), [_frustum_grid_f64(*c) for c in cams], mean_mode)
    assert float((m64 > 0).double().mean()) > 0.2                       # a real share of the grid is sampled
    assert float((m64 == 0).double().mean()) > 0.2                       # ... and a real share is not
    e32 = G.rel_err(got, _to_kernel_order(r32.double(), perm_xzy))
    e64 = G.rel_err(got, _to_kernel_order(r64, perm_xzy))
    G.record("frustum_sample.V%d_mean%d_perm%d" % (V, mean_mode, perm_xzy), "fp32", rel_vs_fp32=e32, rel_vs_f64=e64)
    assert e32 <= FRUSTUM_TOL["fp32"] and e64 <= FRUSTUM_TOL["f64"], (e32, e64)


def _grid_to_lidar():
    X, Y, Z = GRID
    Gm = torch.eye(4)
    Gm[0, 0], Gm[1, 1], Gm[2, 2] = (torch.tensor(PC_MAX) - torch.tensor(PC_MIN)) / torch.tensor([X, Y, Z],
                                                                                             dtype=torch.float32)
    Gm[:3, 3] = torch.tensor(PC_MIN)
    return Gm


@pytest.mark.parametrize("V,mean_mode,perm_xzy", [(1, 1, 0), (2, 1, 1), (3, 0, 0)])
def test_grid_sample_prior_edges(V, mean_mode, perm_xzy):
    """caller grids with coordinates exactly +-1, just outside +-1 and on cell boundaries"""
    g = torch.Generator().manual_seed(20 + V)
    h, w = 12, 40
    X, Y, Z = GRID
    N = X * Y * Z
    depth = torch.randn(V, DN, h, w, generator=g).softmax(1)
    grids = torch.rand(V, N, 3, generator=g) * 2.2 - 1.1
    sizes = torch.tensor([w, h, DN], dtype=torch.float32)
    special = torch.tensor([-1.0, 1.0, -1.0 - 2 ** -20, 1.0 + 2 ** -20, -1.0 + 2 ** -20, 1.0 - 2 ** -20])
    for a in range(3):
        n = 500 * (a + 1)
        grids[:, n:n + 6, a] = special
        # cell boundaries: ((g + 1) * size - 1) / 2 lands on an integer
        k = torch.arange(0, int(sizes[a]), dtype=torch.float32)
        grids[:, n + 6:n + 6 + len(k), a] = (2 * k + 1) / sizes[a] - 1
    out = torch.full((N,), float("nan"), device="cuda")
    assert L().occd_grid_sample_prior_fwd(depth.cuda().data_ptr(), grids.cuda().data_ptr(), V, DN, h, w, X, Y, Z,
                                          mean_mode, out.data_ptr(), perm_xzy, st()) == 0
    got = out.cpu().double()
    gv = [grids[v].view(1, X, Y, Z, 3) for v in range(V)]
    r32, _ = _sample_mean(depth, gv, mean_mode)
    r64, _ = _sample_mean(depth.double(), [t.double() for t in gv], mean_mode)
    e32 = G.rel_err(got, _to_kernel_order(r32.double(), perm_xzy))
    e64 = G.rel_err(got, _to_kernel_order(r64, perm_xzy))
    G.record("grid_sample_prior.V%d_mean%d_perm%d" % (V, mean_mode, perm_xzy), "fp32", rel_vs_fp32=e32,
             rel_vs_f64=e64)
    assert e32 <= GRID_PRIOR_TOL["fp32"] and e64 <= GRID_PRIOR_TOL["f64"], (e32, e64)


# ---- per-image convolution weights ---------------------------------------------------------------------------------
PER_IMAGE_CASES = {
    # id: (B, Cin, Cout, dims, k): positions per image are not multiples of the 128-row tile
    "proj_1x1_b3": (3, 72, 40, (1, 13, 21), (1, 1, 1)),
    "2d_3x3_b2": (2, 32, 48, (1, 11, 19), (1, 3, 3)),
    "3d_3x3x3_b3": (3, 16, 64, (4, 6, 10), (3, 3, 3)),
}


def _per_image_op(case, precision, impl):
    from occdepth_b200 import _lib
    from occdepth_b200.engine import CL, ConvOp, chunk_channels, conv_taps
    B, Cin, Cout, dims, k = PER_IMAGE_CASES[case]
    g = torch.Generator().manual_seed(len(case) + Cin)
    rnd = G.rnd(precision)
    x = rnd(torch.randn(B, Cin, *dims, generator=g))
    ws = [rnd(torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5) for _ in range(B)]
    bias = torch.randn(Cout, generator=g)
    pad = tuple(kk // 2 for kk in k)
    esize = 4 if precision == "tf32" else 2
    Cout_pad, Kpad = -(-Cout // 16) * 16, -(-Cin // chunk_channels(Cin, esize)) * chunk_channels(Cin, esize)
    taps, _ = conv_taps(ws[0], padding=pad)
    wbuf = torch.zeros(B, len(taps), Cout_pad, Kpad)
    for b in range(B):
        for t, wt in enumerate(conv_taps(ws[b], padding=pad)[1]):
            wbuf[b, t, :Cout, :Cin] = wt
    dev = torch.device("cuda")
    wbuf = wbuf.reshape(B * len(taps), Cout_pad, Kpad).to(TDT[precision]).to(dev)
    xin = CL.from_planar(x.to(dev), precision=precision)
    out = CL.alloc(B, *dims, Cout, dev, precision=precision)
    impl_code = {"tc": _lib.CONV_IMPL_TC, "simt": _lib.CONV_IMPL_SIMT, "tcx": _lib.CONV_IMPL_TCX,
                 "halo": _lib.CONV_IMPL_HALO, "halox": _lib.CONV_IMPL_HALOX}[impl]
    op = ConvOp([xin], taps, None, bias.to(dev), dims, out0=out, weight_buf=wbuf, weight_per_image=True,
                impl=impl_code, act="relu", name="per_image_" + case)
    refs = [F.relu(F.conv3d(x[b:b + 1].double(), ws[b].double(), bias.double(), 1, pad)) for b in range(B)]
    return op, out, refs


@PREC
@pytest.mark.parametrize("case,impl", [(c, i) for c in sorted(PER_IMAGE_CASES) for i in ("tc", "simt", "tcx")
                                       if i != "tcx" or PER_IMAGE_CASES[c][4][2] == 3])   # x-packed: three W taps
def test_conv_weight_per_image(case, impl, precision):
    from occdepth_b200 import _lib
    op, out, refs = _per_image_op(case, precision, impl)
    op.run(_lib.stream_ptr())
    torch.cuda.synchronize()
    got = out.to_planar().cpu().double()
    errs = [G.rel_err(got[b:b + 1], refs[b]) for b in range(len(refs))]
    # image 1 through image 0's weights would be far off: the per-image sets are really used
    assert G.rel_err(got[1:2], refs[0]) > 0.1
    G.record("conv_weight_per_image.%s.%s" % (case, impl), precision, rel=max(errs))
    assert max(errs) <= STORE_TOL["conv_per_image"][precision], errs


@pytest.mark.parametrize("impl", ["halo", "halox"])
def test_halo_kernels_refuse_per_image_weights(impl):
    with pytest.raises(RuntimeError, match="per-image"):
        _per_image_op("2d_3x3_b2", "bf16", impl)
