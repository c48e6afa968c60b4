"""Shared GPU parity cases (used by tests/test_gpu_*.py)."""
import torch
import torch.nn.functional as F

from occdepth_b200 import _lib
from occdepth_b200.engine import CL, ConvOp, Plan, conv_taps


def bf16r(t):
    return t.to(torch.bfloat16).float()


def tf32r(t):
    """nearest TF32 value, ties away from zero (cvt.rna.tf32.f32)"""
    return ((t.contiguous().view(torch.int32) + 0x1000) & -0x2000).view(torch.float32)


PRECISIONS = ("tf32", "bf16")
# single-launch tolerance relative to max |reference|: operands are exactly representable, accumulation is fp32, the
# only rounding is the store (bf16: 2^-9, TF32: 2^-11 relative); the bound is 2x that
TOL = {"tf32": 2.0 ** -10, "bf16": 2.0 ** -8}


def rnd(precision):
    return tf32r if precision == "tf32" else bf16r


def report_dir():
    """directory for the measured parity figures (the tolerances in the tests are set to <= 2x what they show):
    $OCCDEPTH_PARITY_DIR, or None -- the tests never write into the source tree"""
    import os
    d = os.environ.get("OCCDEPTH_PARITY_DIR")
    if d:
        os.makedirs(d, exist_ok=True)
    return d


def write_report(name, rep):
    import json
    import os
    d = report_dir()
    if d:
        with open(os.path.join(d, name), "w") as f:
            json.dump(rep, f)


def record(test, precision, **values):
    """append measured parity figures to <report_dir()>/parity_measured.jsonl"""
    import json
    import os
    d = report_dir()
    if d:
        with open(os.path.join(d, "parity_measured.jsonl"), "a") as f:
            f.write(json.dumps(dict(test=test, precision=precision, **values)) + "\n")


def rel_err(got, want):
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-6))


def conv_case(impl, B=1, Cin=32, Cout=32, dims=(6, 10, 12), k=(3, 3, 3), stride=(1, 1, 1), dil=(1, 1, 1),
              pad=None, act="relu", res=False, res_post=False, planar=False, pre=False, seed=0, precision="tf32"):
    """one dense conv through the C ABI vs torch (CPU fp32 on operands rounded to the mode's type). returns rel err."""
    bf16r = rnd(precision)
    g = torch.Generator().manual_seed(seed)
    if pad is None:
        pad = tuple(d * (kk - 1) // 2 for d, kk in zip(dil, k))
    x = bf16r(torch.randn(B, Cin, *dims, generator=g))
    w = bf16r(torch.randn(Cout, Cin, *k, generator=g) / (Cin * k[0] * k[1] * k[2]) ** 0.5)
    b = torch.randn(Cout, generator=g)
    ref = F.conv3d(x, w, b, stride, pad, dil)
    r = None
    if res:
        r = bf16r(torch.randn(ref.shape, generator=g))
    pre_ref = ref + (r if (res and not res_post) else 0)
    actf = {"relu": F.relu, "none": lambda t: t, "silu": F.silu, "sigmoid": torch.sigmoid,
            "leaky": lambda t: F.leaky_relu(t, 0.01)}[act]
    out_ref = actf(pre_ref) + (r if (res and res_post) else 0)
    dev = torch.device("cuda")
    plan = Plan(dev, precision=precision)
    xin = CL.from_planar(x.to(dev), precision=precision)
    rcl = CL.from_planar(r.to(dev), precision=precision) if res else None
    out1, mode = None, "none"
    od = tuple(ref.shape[2:])
    if planar:
        out1, mode = torch.zeros(B, Cout + 3, *od, device=dev), "planar"
    elif pre:
        out1, mode = plan.alloc(B, od[0], od[1], od[2], Cout), "cl"
    y = plan.conv(xin, w.to(dev), b.to(dev), stride=stride, padding=pad, dilation=dil, act=act,
                  res1=None if res_post else rcl, res2=rcl if res_post else None, res2_post=res_post,
                  out1=out1, out1_mode=mode, out1_coff=2 if planar else 0, impl=impl,
                  out=plan.alloc(B, od[0], od[1], od[2], Cout))
    plan.run()
    torch.cuda.synchronize()
    errs = [rel_err(y.to_planar().cpu(), out_ref)]
    if planar:
        errs.append(rel_err(out1[:, 2:2 + Cout].cpu(), pre_ref))
        assert float(out1[:, :2].abs().max()) == 0 and float(out1[:, 2 + Cout:].abs().max()) == 0
    elif pre:
        errs.append(rel_err(out1.to_planar().cpu(), pre_ref))
    return max(errs), plan.ops[0].info()


def convT_case(impl, Cin=32, Cout=16, dims=(4, 6, 5), seed=0, skip=True, precision="tf32"):
    bf16r = rnd(precision)
    g = torch.Generator().manual_seed(seed)
    x = bf16r(torch.randn(1, Cin, *dims, generator=g))
    w = bf16r(torch.randn(Cin, Cout, 3, 3, 3, generator=g) / (Cin * 8) ** 0.5)
    b = torch.randn(Cout, generator=g)
    ref = F.relu(F.conv_transpose3d(x, w, b, 2, 1, 1))
    sk = bf16r(torch.randn(ref.shape, generator=g))
    if skip:
        ref = ref + sk
    dev = torch.device("cuda")
    plan = Plan(dev, precision=precision)
    y = plan.conv_transpose_k3s2(CL.from_planar(x.to(dev), precision=precision), w.to(dev), b.to(dev), act="relu",
                                 res_post=CL.from_planar(sk.to(dev), precision=precision) if skip else None,
                                 impl=impl)
    plan.run()
    torch.cuda.synchronize()
    return rel_err(y.to_planar().cpu(), ref), plan.ops[0].info()


def multi_case(impl, C=32, dims=(6, 8, 8), seed=0, precision="tf32"):
    """the fused ASPP conv2 stage: three sources, dilations 1/2/3, one accumulator, residual + relu."""
    bf16r = rnd(precision)
    g = torch.Generator().manual_seed(seed)
    xs = [bf16r(torch.randn(1, C, *dims, generator=g)) for _ in range(3)]
    ws = [bf16r(torch.randn(C, C, 3, 3, 3, generator=g) / (C * 27) ** 0.5) for _ in range(3)]
    b = torch.randn(C, generator=g)
    r = bf16r(torch.randn(1, C, *dims, generator=g))
    ref = sum(F.conv3d(x, w, None, 1, d, d) for x, w, d in zip(xs, ws, (1, 2, 3)))
    ref = F.relu(ref + b.view(1, -1, 1, 1, 1) + r)
    dev = torch.device("cuda")
    plan = Plan(dev, precision=precision)
    y = plan.conv_multi([CL.from_planar(x.to(dev), precision=precision) for x in xs], [w.to(dev) for w in ws],
                        b.to(dev), [1, 2, 3], [1, 2, 3], act="relu",
                        res1=CL.from_planar(r.to(dev), precision=precision), impl=impl)
    plan.run()
    torch.cuda.synchronize()
    return rel_err(y.to_planar().cpu(), ref), plan.ops[0].info()


CONV_CASES = {
    "k1_c32": dict(k=(1, 1, 1), Cin=32, Cout=32),
    "k3_c32_d1": dict(),
    "k3_c32_d2": dict(dil=(2, 2, 2)),
    "k3_c32_d3_res": dict(dil=(3, 3, 3), res=True),
    "k3_c64_co80": dict(Cin=64, Cout=80, pre=True),
    "k3_c16": dict(Cin=16, Cout=16),
    "k3_c96_co20_planar": dict(Cin=96, Cout=20, planar=True, act="none"),
    "k3_c200_co200": dict(Cin=200, Cout=200, dims=(4, 5, 6)),
    "k3_c34_co2": dict(Cin=34, Cout=2, act="none", planar=True),
    "k113_s2": dict(k=(1, 1, 3), stride=(1, 1, 2), Cin=16, Cout=16),
    "k3_s2_co320": dict(stride=(2, 2, 2), pad=(1, 1, 1), Cin=64, Cout=320, dims=(8, 8, 6)),
    "2d_k3_c163": dict(k=(1, 3, 3), Cin=163, Cout=80, dims=(1, 23, 37), act="leaky"),
    "2d_k1_c3_silu": dict(k=(1, 1, 1), Cin=3, Cout=64, dims=(1, 19, 33), act="silu"),
    "k222_s2_pool": dict(k=(2, 2, 2), stride=(2, 2, 2), pad=(0, 0, 0), Cin=64, Cout=128, act="none"),
    "k1_sigmoid_b2": dict(B=2, k=(1, 1, 1), Cin=256, Cout=512, dims=(4, 4, 2), act="sigmoid", planar=True),
    "k3_respost": dict(res=True, res_post=True),
}


HALO_CASES = {
    "h_c32_d1": dict(Cin=32, Cout=32, dims=(6, 10, 12)),
    "h_c32_d2": dict(Cin=32, Cout=32, dims=(9, 11, 14), dil=(2, 2, 2)),
    "h_c32_d3_res": dict(Cin=32, Cout=32, dims=(8, 13, 32), dil=(3, 3, 3), res=True),
    "h_c16_n16": dict(Cin=16, Cout=16, dims=(5, 9, 16)),
    "h_c64_n32_pre": dict(Cin=64, Cout=32, dims=(6, 9, 20), pre=True),
    "h_c32_n2_planar": dict(Cin=32, Cout=2, dims=(6, 10, 32), act="none", planar=True),
    "h_2d_c48": dict(k=(1, 3, 3), Cin=48, Cout=40, dims=(1, 21, 70), act="leaky"),
    "h_2d_b2_res": dict(B=2, k=(1, 3, 3), Cin=32, Cout=32, dims=(1, 12, 40), res=True),
    "h_3d_b3": dict(B=3, Cin=16, Cout=32, dims=(4, 6, 8)),
    "h_big": dict(Cin=32, Cout=32, dims=(20, 40, 32), dil=(1, 1, 1)),
    "h_big_d3": dict(Cin=32, Cout=32, dims=(20, 40, 32), dil=(3, 3, 3)),
}
