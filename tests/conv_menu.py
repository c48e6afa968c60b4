"""The compiled convolution menu and the cases that reach every entry of it under tests/conv_replay.py's float64
comparator.  Shared by tests/test_gpu_conv_menu.py and tests/test_conv_menu_host.py (a plain helper, imported like
gpu_cases).

  parse_menu()        the N tiles of each kernel (the NTiles<...> lists of csrc/conv_kernels.cuh) and kPingPongMaxN,
                      read from the source, so that a tile added to the menu is a cell no case reaches yet
  compiled_cells()    every (precision, kernel, N tile, schedule) instantiation: conv_tc_kernel<T, N, XP, PP> (tc,
                      tcx) and conv_halox_kernel<T, N, PP> with PP only for N <= kPingPongMaxN, conv_halo_kernel<T, N>
                      (cooperative only), and the SIMT kernel
  FAMILIES            name -> build(precision, device, simt) -> [(ConvOp, expected info fields)].  Each case plans a
                      ConvOp directly with a forced impl=, on the buffers and windows it describes; the values are
                      written later by conv_replay.fill.  simt=True plans every case on the SIMT kernel instead (the
                      only one that plans without a driver) and drops the tensor-core expectations.
  refusals()          name -> (build(precision, device), exception, words of its message): descriptors the planner
                      must refuse
"""
import os
import re

import torch

import gpu_cases as G
from occdepth_b200 import _lib
from occdepth_b200.engine import CL, ConvOp, Plan, chunk_channels, conv_taps, out_size

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS_CUH = os.path.join(ROOT, "occdepth_b200", "csrc", "conv_kernels.cuh")
IMPL = {"tc": _lib.CONV_IMPL_TC, "tcx": _lib.CONV_IMPL_TCX, "halo": _lib.CONV_IMPL_HALO,
        "halox": _lib.CONV_IMPL_HALOX, "simt": _lib.CONV_IMPL_SIMT}
TC_KERNELS = ("tc", "tcx", "halo", "halox")
ACTS = ("none", "relu", "leaky", "silu", "sigmoid")
CLASS_MODES = ("classes", "classes_conf", "classes_probs")
MODE_NUM = {"classes": _lib.OUT1_CLASS_U16, "classes_conf": _lib.OUT1_CLASS_U16_CONF,
            "classes_probs": _lib.OUT1_CLASS_U16_PROBS}
LUT = tuple((7 * i + 3) % 251 for i in range(20))         # a label remap of the 20-class cases


def _round_up(a, b):
    return (a + b - 1) // b * b


# ---------------------------------------------------------------------------------------------------------------
def parse_menu(path=KERNELS_CUH):
    """-> ({kernel: set of N tiles}, kPingPongMaxN) from `using <Kernel>Tiles = NTiles<...>;` and the constant"""
    with open(path) as f:
        src = f.read()
    menu = {name.lower(): {int(n) for n in ns.split(",")}
            for name, ns in re.findall(r"using\s+(\w+)Tiles\s*=\s*NTiles<([^>]*)>", src)}
    pp_max = int(re.search(r"constexpr\s+int\s+kPingPongMaxN\s*=\s*(\d+)\s*;", src).group(1))
    return menu, pp_max


def compiled_cells():
    menu, pp_max = parse_menu()
    cells = set()
    for p in G.PRECISIONS:
        cells.add((p, "simt", 0, "none"))
        for kern, tiles in menu.items():
            for n in tiles:
                cells.add((p, kern, n, "cooperative"))
                if kern != "halo" and n <= pp_max:
                    cells.add((p, kern, n, "pingpong"))
    return cells


# ---------------------------------------------------------------------------------------------------------------
def _cl(dev, precision, B, D, H, W, C, coff=0, extra=0, margin=0):
    """a channel window [coff, coff + C) of a zero buffer `extra` channels wider, with `margin` planes each side"""
    dt = torch.float32 if precision == "tf32" else torch.bfloat16
    buf = torch.zeros(B, D + 2 * margin, H, W, _round_up(coff + C, 8) + extra, dtype=dt, device=dev)
    return CL(buf, C, coff, margin, D)


def conv_op(dev, precision, impl, B=1, Cin=32, Cout=32, dims=(6, 10, 12), k=(3, 3, 3), stride=(1, 1, 1),
            dil=(1, 1, 1), pad=None, act="relu", res=False, res_post=False, res_both=False, planar=False, pre=False,
            exact=False, margin=0, windows=False, cls=None, lut=None, per_image=False, seed=0):
    """one dense conv (gpu_cases.conv_case's arguments) as a ConvOp on kernel `impl`.  res: a residual, before the
    activation (res1) or after it (res2, res_post); res_both: res1 and a res2 (res_post: after the activation);
    planar: fp32 planar out1 at out1_coff 3; pre: channels-last out1; exact: out0_exact; margin: planes of source data
    each side of D (src_d0); windows: every channels-last operand a window at a non-zero offset of a wider buffer;
    cls: a class-map mode (no out0) with label remap lut; per_image: B run-time weight sets"""
    g = torch.Generator().manual_seed(seed)
    if pad is None:
        pad = tuple(d * (kk - 1) // 2 for d, kk in zip(dil, k))
    od = tuple(out_size(dims[i], k[i], stride[i], pad[i], dil[i]) for i in range(3))
    win = dict(coff=8, extra=16) if windows else {}
    x = _cl(dev, precision, B, *dims, Cin, margin=margin, **win)
    w = torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5
    bias = torch.randn(Cout, generator=g).to(dev)
    taps, ws = conv_taps(w.to(dev), dil, pad)

    def cl_out(C, i=0):
        return _cl(dev, precision, B, *od, C, coff=8 * (i + 1), extra=8) if windows else _cl(dev, precision, B, *od, C)
    kw = dict(act=act, stride=stride, impl=impl, name="menu", out0_exact=exact, lut=lut)
    if cls is None:
        kw["out0"] = cl_out(Cout)
    else:
        rows = {"classes": (B,), "classes_conf": (2, B), "classes_probs": ((1 + Cout) * B,)}[cls]
        kw.update(out1=torch.zeros(rows + od, dtype=torch.uint16, device=dev), out1_mode=cls)
    if res_both:
        kw.update(res1=cl_out(Cout, 1), res2=cl_out(Cout, 2), res2_post=res_post)
    elif res:
        kw["res2" if res_post else "res1"] = cl_out(Cout, 1)
        kw["res2_post"] = res_post
    if planar:
        kw.update(out1=torch.zeros((B, Cout + 5) + od, device=dev), out1_mode="planar", out1_coff=3)
    elif pre:
        kw.update(out1=cl_out(Cout, 3), out1_mode="cl")
    if per_image:
        esize = 4 if precision == "tf32" else 2
        kw.update(weight_per_image=True,
                  weight_buf=torch.zeros(B * len(taps), _round_up(Cout, 16), _round_up(Cin, chunk_channels(Cin, esize)),
                                         dtype=x.buf.dtype, device=dev))
    return ConvOp([x], taps, ws, bias, od, **kw)


def multi_op(dev, precision, impl, Cs=(48, 24, 20), Cout=20, dims=(4, 7, 9), seed=0):
    """three sources of unequal C (the last not a multiple of the K chunk), each a window of a wider buffer, with
    dilations 1 / 2 / 3, one accumulator, a residual before the relu"""
    g = torch.Generator().manual_seed(seed)
    srcs = [_cl(dev, precision, 1, *dims, C, coff=8 * i, extra=8) for i, C in enumerate(Cs)]
    taps, ws = [], []
    for i, C in enumerate(Cs):
        w = (torch.randn(Cout, C, 3, 3, 3, generator=g) / (27 * C) ** 0.5).to(dev)
        t, wl = conv_taps(w, (i + 1,) * 3, (i + 1,) * 3, src=i)
        taps += t
        ws += wl
    bias = torch.randn(Cout, generator=g).to(dev)
    return ConvOp(srcs, taps, ws, bias, dims, out0=_cl(dev, precision, 1, *dims, Cout, coff=16, extra=8), act="relu",
                  res1=_cl(dev, precision, 1, *dims, Cout, coff=8), impl=impl, name="menu.multi")


def convT_ops(dev, precision, impl, Cin=32, Cout=16, dims=(4, 6, 5), seed=0):
    """ConvTranspose3d(k3, s2) + relu + skip: on the per-tap kernel one launch of 8 tap groups, else 8 launches"""
    g = torch.Generator().manual_seed(seed)
    plan = Plan(dev, precision=precision)
    x = _cl(dev, precision, 1, *dims, Cin)
    skip = _cl(dev, precision, 1, *(2 * d for d in dims), Cout)
    w = (torch.randn(Cin, Cout, 3, 3, 3, generator=g) / (Cin * 8) ** 0.5).to(dev)
    plan.conv_transpose_k3s2(x, w, torch.randn(Cout, generator=g).to(dev), act="relu", res_post=skip, impl=impl)
    return plan.ops


# ---------------------------------------------------------------------------------------------------------------
# families: name -> build(precision, dev, simt) -> [(op, expect)]
def _dense(kern, simt, expect=None, **kw):
    return lambda p, dev: (conv_op(dev, p, IMPL["simt" if simt else kern], **kw), {} if simt else (expect or {}))


def _ntiles(simt):
    import test_gpu_conv_ntiles as NT
    cases = []
    for kern, lst in NT.CASES.items():
        for Cout, kw in lst:
            n = 3 * _round_up(Cout, 16) if kern in ("tcx", "halox") else Cout
            cases.append(_dense(kern, simt, dict(N_tile=n), Cout=Cout, act="leaky", **kw))
    return cases


def _pingpong(simt):
    import test_gpu_conv_pingpong as PP
    cases = []
    for name in sorted(PP.CASES):
        kern, kw, n_tile, n_tiles = PP.CASES[name]
        ex = dict(schedule="pingpong", N_tile=n_tile)
        if n_tiles is not None:
            ex.update(grid_y=n_tiles, grid_x=min(n_tiles, 132))
        cases.append(_dense(kern, simt, ex, **kw))
    kern, kw, n_tile, n_tiles = PP.SMALL
    cases.append(_dense(kern, simt, dict(schedule="cooperative", N_tile=n_tile, grid_y=n_tiles), **kw))
    cases.append(_dense("tc", simt, dict(schedule="cooperative", N_tile=160), Cin=64, Cout=160, dims=(8, 80, 128)))
    cases.append(_dense("tc", simt, dict(schedule="cooperative"), k=(1, 1, 1), Cin=32, Cout=64, dims=(1, 330, 512)))
    return cases


def _conv_cases(simt):
    return [_dense("tc", simt, None, **G.CONV_CASES[name]) for name in sorted(G.CONV_CASES)]


def _halo_cases(simt):
    cases = []
    for name in sorted(G.HALO_CASES):
        kw = G.HALO_CASES[name]

        def build(p, dev, kw=kw, name=name):
            # one K chunk of resident weights; a TF32 W = 32 box of 27 resident taps does not fit (gpu_cases)
            if kw.get("Cin", 32) > (32 if p == "tf32" else 64) or (p == "tf32" and name == "h_big"):
                return None
            return _dense("halo", simt, None, **kw)(p, dev)
        cases.append(build)
    return cases


def _rb(simt):
    """each tensor-core kernel at every K-chunk row width: Cin = rb / element size"""
    shapes = {"tc": dict(Cout=24, dims=(5, 9, 13)), "tcx": dict(k=(1, 3, 3), Cout=32, dims=(2, 9, 40)),
              "halo": dict(Cout=32, dims=(5, 9, 13)), "halox": dict(Cout=32, dims=(8, 16, 32))}
    cases = []
    for kern in TC_KERNELS:
        for rb in (32, 64, 128):
            def build(p, dev, kern=kern, rb=rb):
                Cin = rb // (4 if p == "tf32" else 2)
                return _dense(kern, simt, dict(KC=Cin), Cin=Cin, act="relu", **shapes[kern])(p, dev)
            cases.append(build)
    return cases


CLASS_SHAPES = {"simt": dict(B=2, Cin=32, dims=(5, 9, 13)),
                "tc": dict(B=2, Cin=32, dims=(4, 40, 64)),
                "tcx": dict(B=2, k=(1, 3, 3), Cin=40, dims=(1, 24, 70)),
                "halo": dict(B=2, Cin=32, dims=(5, 9, 13)),
                "halox": dict(B=2, Cin=32, dims=(4, 12, 32))}


def _classes(simt):
    cases = []
    for kern, shape in CLASS_SHAPES.items():
        for mode in CLASS_MODES:
            for lut in (None, LUT):
                cases.append(_dense(kern, simt, None, Cout=20, cls=mode, lut=lut, act="none", **shape))
    # the x-packed kernels write the probabilities at N = 240 (3 x 80 channels): no kProbsMaxN for them (and no lut:
    # it holds at most 64 labels)
    for kern in ("tcx", "halox"):
        cases.append(_dense(kern, simt, dict(N_tile=240), Cout=75, cls="classes_probs", act="none",
                            **dict(CLASS_SHAPES[kern], k=(1, 3, 3))))
    # a per-tap N tile of 112 writes the map (the probabilities are refused: REFUSALS)
    cases.append(_dense("tc", simt, dict(N_tile=112), Cout=100, cls="classes", Cin=32, dims=(4, 40, 128), act="none"))
    return cases


def _epilogue(simt):
    """the per-tap kernel's epilogue variants: every activation through the fast row epilogue (out0 and one
    residual) and the general one (a channels-last out1 and both residuals, every operand a channel window); the
    residual placements, out0_exact, planar out1 at a channel offset, Cout not a multiple of 8"""
    base = dict(B=2, Cin=24, Cout=20, dims=(3, 7, 45))
    cases = []
    for act in ACTS:
        cases.append(_dense("tc", simt, None, act=act, res=True, **base))
        cases.append(_dense("tc", simt, None, act=act, res_both=True, pre=True, windows=True, **base))
    cases += [_dense("tc", simt, None, act="silu", res=True, res_post=True, **base),
              _dense("tc", simt, None, act="leaky", res_both=True, res_post=True, **base),
              _dense("tc", simt, None, act="relu", res=True, exact=True, windows=True, **base),
              _dense("tc", simt, None, act="sigmoid", planar=True, **base),
              _dense("tc", simt, None, act="relu", B=1, Cin=24, Cout=2, dims=(3, 7, 45), windows=True)]
    return cases


def _windows_margins(simt):
    """source margin planes (src_d0 > 0) holding data, and channel windows, on the kernels that take them"""
    return [_dense("tc", simt, None, margin=2, windows=True, res=True, Cin=40, Cout=20, dims=(5, 9, 13)),
            _dense("tc", simt, None, margin=1, stride=(2, 2, 2), Cin=32, Cout=24, dims=(6, 9, 13)),
            _dense("tcx", simt, None, margin=2, windows=True, Cin=24, Cout=20, dims=(4, 9, 40)),
            _dense("halo", simt, None, margin=2, windows=True, res=True, Cin=32, Cout=20, dims=(5, 9, 13)),
            _dense("halox", simt, None, margin=2, windows=True, res=True, Cin=32, Cout=20, dims=(6, 12, 16)),
            _dense("halox", simt, None, margin=3, dil=(3, 3, 3), Cin=16, Cout=16, dims=(7, 10, 8))]


def _sources_groups_weights(simt):
    cases = [lambda p, dev: (multi_op(dev, p, IMPL["simt" if simt else "tc"]), {})]

    def convT(p, dev):
        ops = convT_ops(dev, p, IMPL["simt" if simt else "tc"])
        assert simt or (len(ops) == 1 and ops[0].desc.n_groups == 8), len(ops)
        return [(op, {}) for op in ops]
    cases.append(convT)
    for kern, kw in (("tc", dict(Cin=40, Cout=24, dims=(3, 7, 45))), ("simt", dict(Cin=40, Cout=24, dims=(3, 7, 9))),
                     ("tcx", dict(k=(1, 3, 3), Cin=40, Cout=32, dims=(1, 9, 70)))):
        cases.append(_dense(kern, simt, None, B=2, per_image=True, act="relu", **kw))
    return cases


def _edges(simt):
    """extents that are no multiple of the tile box, several items, a single M tile, fewer tiles than SMs, and a
    tail wave of one tile past one and two multiples of the grid"""
    cases = []
    for kern, kw in (("tc", dict(dims=(5, 9, 13))), ("tcx", dict(k=(1, 3, 3), dims=(1, 11, 61))),
                     ("halo", dict(dims=(5, 9, 13))), ("halox", dict(dims=(5, 9, 16))), ("simt", dict(dims=(5, 9, 13)))):
        cases.append(_dense(kern, simt, None, B=3, Cin=32, Cout=20, res=True, **kw))
    for kern, kw in (("tc", dict(dims=(1, 4, 8))), ("tcx", dict(k=(1, 3, 3), dims=(1, 3, 20))),
                     ("halo", dict(dims=(2, 3, 8))), ("halox", dict(dims=(2, 3, 8)))):
        ex = dict(grid_x=1) if kern in ("tc", "tcx") else {}
        cases.append(_dense(kern, simt, ex, Cin=32, Cout=16, **kw))
    for rows in (133, 265):
        cases.append(_dense("tc", simt, dict(grid_x=132, grid_y=rows, N_tile=16), k=(1, 1, 1), Cin=32, Cout=16,
                            dims=(1, rows, 128), res=True))
    return cases


FAMILY_CASES = {"ntiles": _ntiles, "pingpong": _pingpong, "conv_cases": _conv_cases, "halo_cases": _halo_cases,
                "rb": _rb, "classes": _classes, "epilogue": _epilogue, "windows_margins": _windows_margins,
                "sources_groups_weights": _sources_groups_weights, "edges": _edges}
FAMILIES = sorted(FAMILY_CASES)


def build(family, precision, dev, simt=False):
    """-> [(ConvOp, expected info fields)] of one family"""
    out = []
    for case in FAMILY_CASES[family](simt):
        r = case(precision, dev)
        if r is None:
            continue
        out += r if isinstance(r, list) else [r]
    return out


# ---------------------------------------------------------------------------------------------------------------
# what the planner must refuse: name -> (build(precision, dev), exception type, words of the message)
def refusals():
    from occdepth_b200.engine import ClassMapUnsupported
    r = {"probs_tc_n112": (lambda p, dev: conv_op(dev, p, IMPL["tc"], Cout=100, cls="classes_probs", Cin=32,
                                                   dims=(4, 40, 128), act="none"),
                           ClassMapUnsupported, "at most 96")}
    for kern in ("halo", "halox"):
        r["per_image_" + kern] = (lambda p, dev, kern=kern: conv_op(dev, p, IMPL[kern], B=2, per_image=True, Cin=32,
                                                                     Cout=32, dims=(2, 8, 16)),
                                  RuntimeError, "per-image weights")
    return r
