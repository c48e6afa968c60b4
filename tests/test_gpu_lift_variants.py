"""SFA lift (`occd_sfa_lift_fwd`) called directly, across its launch variants, against a float64 restatement.

Each case reaches one instantiation of the kernel: element type x view count x (NV, G) lane layout x kernel (the
P == 1 fast path or the general one).  The cases together reach every instantiation `launch_nv` picks by default
(test_cases_cover_the_default_menu); the other factors -- output mode, scales and floor divisors, view strides,
prior, NYU permutation, voxel counts that do not fill the last block -- vary across them.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import gpu_cases as G
import launch_replay as LR

# bounds relative to max |ref|: twice the largest figure measured on an H100 (OCCDEPTH_PARITY_DIR), never looser than
# the one-store bound G.TOL for rounded outputs.  fp32 outputs differ from the reference only in operation order.
TOL = {"f32_planar": 4e-7, "f32_cl": 3.6e-7, "tf32_cl": 8e-4, "bf16_cl": G.TOL["bf16"]}
SENTINEL = -448.0         # exact in bf16 and TF32: pad channels of channels-last outputs must keep it
VEC = {"f32": 4, "bf16": 8}
OUT_MODES = ("f32_planar", "bf16_cl", "f32_cl", "tf32_cl")
DIVS = (1, 2, 3, 4, 6, 8)
IMG_H, IMG_W = 29, 43


# ---- the instantiation a call reaches: the rule of launch_nv / launch_g (csrc/sfa_lift.cu) ----------------------------
def lane_layout(dtype, C_):
    """(NV, G): 16-byte vectors per lane and lanes per voxel (OCCD_LIFT_NV unset)"""
    vecs = -(-C_ // VEC[dtype])
    if vecs <= 4:
        return 1, 4
    nv = 2 if dtype == "bf16" else 4
    lanes = (4, 8, 16, 32) if dtype == "bf16" else (2, 4, 8, 16)
    for lim, g in zip((8, 16, 32, 64), lanes):
        if vecs <= lim:
            return nv, g
    raise ValueError("C too large")


def general_smem(V, G_, P):
    """bytes of index staging of the general kernel: launch_g refuses more than 200 KiB"""
    return V * (256 // G_) * 4 * P * 17


def instantiation(case):
    return (case["dtype"], case["V"], lane_layout(case["dtype"], case["C"]), "p1" if case["P"] == 1 else "general")


def default_menu():
    layouts = {"f32": [(1, 4), (4, 2), (4, 4), (4, 8), (4, 16)], "bf16": [(1, 4), (2, 4), (2, 8), (2, 16), (2, 32)]}
    return {(dt, V, lay, k) for dt in VEC for V in (1, 2, 3, 4) for lay in layouts[dt] for k in ("p1", "general")}


# ---- cases --------------------------------------------------------------------------------------------------------
def _cases():
    chans = {"f32": (16, 32, 64, 128, 256), "bf16": (32, 64, 128, 256, 512)}
    cases, i = [], 0
    for dt in ("f32", "bf16"):
        for V in (1, 2, 3, 4):
            for C_ in chans[dt]:
                for kern in ("p1", "general"):
                    cases.append(_case(i, dt, V, C_, kern))
                    i += 1
    # partial lane widths: the last lane group of a voxel holds fewer vectors than the others
    for dt, C_, V in (("f32", 36, 2), ("f32", 196, 3), ("bf16", 72, 4), ("bf16", 392, 2)):
        for kern in ("p1", "general"):
            cases.append(_case(i, dt, V, C_, kern))
            i += 1
    return cases


def _case(i, dt, V, C_, kern):
    ns = 1 + (i // 2) % 4
    P = 1 if kern == "p1" else (5, 9)[(i // 2) % 2]
    if general_smem(V, lane_layout(dt, C_)[1], P) > 200 * 1024:
        P = 5
    return dict(
        id="%s_V%d_C%d_%s_%d" % (dt, V, C_, kern, i), dtype=dt, V=V, C=C_, P=P,
        out_mode=OUT_MODES[(i + i // 8) % 4],
        divs=[DIVS[(i // 2 + s) % 6] for s in range(ns)],
        padded_views=(i % 3 == 0), prior=(i % 5 in (1, 3)), nyu=(i % 4 in (1, 2)),
        grid=((5, 7, 9), (3, 11, 13), (4, 5, 6))[i % 3], seed=i)


CASES = _cases()


# ---- float64 restatement of the lift: launch_replay.lift_ref -----------------------------------------------------------
lift_ref = LR.lift_ref


def make_inputs(case):
    g = torch.Generator().manual_seed(1000 + case["seed"])
    V, C_, P = case["V"], case["C"], case["P"]
    X, S1, S2 = case["grid"]
    N = X * S1 * S2
    # pixels up to a few outside the image (negative ones too: floor, not truncation, for divisors 3 and 6); points
    # outside the image may still be flagged in FOV: their index can fall outside a scale's map
    x = torch.randint(-5, IMG_W + 5, (V, N, P), generator=g)
    y = torch.randint(-4, IMG_H + 4, (V, N, P), generator=g)
    fov = torch.rand(V, N, P, generator=g) < 0.8
    pix = torch.stack([x, y], -1)
    feats = []
    for d in case["divs"]:
        h, w = -(-IMG_H // d), -(-IMG_W // d)
        f = torch.randn(V, h, w, C_, generator=g)
        feats.append(G.bf16r(f) if case["dtype"] == "bf16" else f)
    prior = torch.rand(N, generator=g) * 2 if case["prior"] else None
    return feats, pix, fov, prior


def run_lift(feats, divs, pix, fov, dtype, out_mode, out_cstride=None, perm=None, prior=None, scale_const=1.0,
             padded_views=False):
    """feats: per scale [V, h, w, C] float; returns the raw output buffer (planar [C][N] or [N][cstride])"""
    from occdepth_b200 import _lib
    V, N, P, _ = pix.shape
    C_ = feats[0].shape[3]
    tdt = torch.float32 if dtype == "f32" else torch.bfloat16
    p = _lib.SfaParams()
    keep = []
    for s, (f, d) in enumerate(zip(feats, divs)):
        h, w = f.shape[1], f.shape[2]
        dense = h * w * C_
        vs = dense + (3 * C_ if padded_views else 0)
        # views inside a larger buffer: the gap between them is NaN, so a read through the wrong stride shows up
        buf = torch.full((V, vs), float("nan"), dtype=tdt)
        buf[:, :dense] = f.reshape(V, dense).to(tdt)
        buf = buf.cuda()
        keep.append(buf)
        p.feat[s], p.h[s], p.w[s], p.div[s] = buf.data_ptr(), h, w, d
        p.vstride[s] = vs if padded_views else 0
    p.n_scales, p.n_views, p.C = len(feats), V, C_
    p.feat_dtype = _lib.DTYPE_F32 if dtype == "f32" else _lib.DTYPE_BF16
    pix_d, fov_d = pix.contiguous().cuda(), fov.contiguous().cuda()
    p.pix, p.fov, p.N, p.P = pix_d.data_ptr(), fov_d.data_ptr(), N, P
    mode = {"f32_planar": _lib.SFA_OUT_F32_PLANAR, "bf16_cl": _lib.SFA_OUT_BF16_CL, "f32_cl": _lib.SFA_OUT_F32_CL,
            "tf32_cl": _lib.SFA_OUT_TF32_CL}[out_mode]
    if out_mode == "f32_planar":
        out = torch.full((C_, max(N, 1)), float("nan"), device="cuda")
        cst = C_
    else:
        cst = out_cstride or C_
        out = torch.full((max(N, 1), cst), SENTINEL, device="cuda",
                         dtype=torch.bfloat16 if out_mode == "bf16_cl" else torch.float32)
    p.out, p.out_mode, p.out_cstride = out.data_ptr(), mode, cst
    if perm is not None:
        p.perm_nyu, p.S1, p.S2 = 1, perm[0], perm[1]
    if prior is not None:
        prior_d = prior.float().cuda()
        keep.append(prior_d)
        p.prior, p.scale_const = prior_d.data_ptr(), float(scale_const)
    rc = _lib.lib().occd_sfa_lift_fwd(C.byref(p), _lib.stream_ptr())
    torch.cuda.synchronize()
    return rc, out.float().cpu()


def check_output(out, ref, out_mode, C_, tag, precision_label):
    """compares a run_lift buffer with the [N, C] float64 reference and records the relative error"""
    if out_mode == "f32_planar":
        got = out.t()
    else:
        got = out[:, :C_]
        assert torch.all(out[:, C_:] == SENTINEL), "pad channels written"
    assert not torch.isnan(got).any(), "output not written everywhere"
    err = G.rel_err(got.double(), ref)
    G.record("lift_variants." + tag, precision_label, out_mode=out_mode, rel=err)
    if out_mode == "tf32_cl":
        assert torch.equal(got, G.tf32r(got)), "TF32_CL output holds non-TF32 values"
    assert err <= TOL[out_mode], err


def _perm_of(case):
    X, S1, S2 = case["grid"]
    return (S1, S2) if case["nyu"] else None


# ---- tests --------------------------------------------------------------------------------------------------------
def test_cases_cover_the_default_menu():
    """every default (dtype, V, NV, G) instantiation of both kernels is reached by some case, and nothing else is"""
    reached = {instantiation(c) for c in CASES}
    assert reached == default_menu()
    assert len(default_menu()) == 2 * 4 * 5 * 2
    # the other factors take every value in both element types and both kernels
    for dt in VEC:
        for kern in ("p1", "general"):
            sub = [c for c in CASES if c["dtype"] == dt and (c["P"] == 1) == (kern == "p1")]
            assert {c["out_mode"] for c in sub} == set(OUT_MODES)
            assert {len(c["divs"]) for c in sub} == {1, 2, 3, 4}
            assert {d for c in sub for d in c["divs"]} == set(DIVS)
            for key in ("padded_views", "prior", "nyu"):
                assert {c[key] for c in sub} == {False, True}
            assert all(c["grid"][0] * c["grid"][1] * c["grid"][2] % 32 for c in sub)


def test_reference_restatement_matches_oracle():
    """the float64 restatement agrees with the oracle's SFA / multi-scale lift on cases the oracle supports (every
    in-FOV point inside every map)"""
    from oracle import functional as OF
    from synthetic import random_indices
    g = torch.Generator().manual_seed(7)
    for dataset, V, P, scales in (("kitti", 2, 1, (1, 2)), ("NYU", 3, 5, (1, 2, 4)), ("kitti", 1, 9, (1,))):
        scene, ps = (12, 10, 8), 2
        S = [s // ps for s in scene]
        N = S[0] * S[1] * S[2]
        C_ = 12
        H, W = 16, 24
        pix, fov = random_indices(N, W, H, n_views=V, P=P, seed=V + P, margin=(4, 3))
        x_rgb = [{} for _ in range(V)]
        feats = []
        for s in scales:
            f = torch.randn(V, C_, H // s, W // s, generator=g, dtype=torch.float64)
            feats.append(f.permute(0, 2, 3, 1))
            for v in range(V):
                x_rgb[v]["1_%d" % s] = f[v]
        want = OF.lift_flosp(x_rgb, pix, fov, [str(s) for s in scales], scene, dataset, ps)     # (C, X, Y, Z)
        perm = (S[1], S[2]) if dataset == "NYU" else None
        got = lift_ref(feats, scales, pix, fov, perm=perm)
        assert float((got.t().reshape(want.shape) - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_lift_variant(case):
    feats, pix, fov, prior = make_inputs(case)
    perm = _perm_of(case)
    ref = lift_ref([f.double() for f in feats], case["divs"], pix, fov, perm=perm, prior=prior, scale_const=100.0)
    rc, out = run_lift(feats, case["divs"], pix, fov, case["dtype"], case["out_mode"], out_cstride=case["C"] + 8,
                       perm=perm, prior=prior, scale_const=100.0, padded_views=case["padded_views"])
    assert rc == 0
    assert fov.float().mean() > 0.5
    check_output(out, ref, case["out_mode"], case["C"], case["id"], case["dtype"])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("P", [1, 5])
def test_lift_edge_inputs(dtype, P):
    """masked views, a near-zero feature vector, negative coordinates under floor division, in-FOV indices outside the
    map, and |x| > 2^30 -- each on its own voxels of one V = 2 launch"""
    g = torch.Generator().manual_seed(5 + P)
    V, C_, N = 2, 32, 200
    h, w = 10, 14
    f = torch.randn(V, h, w, C_, generator=g)
    f[0, 2, 3] = 1e-10 * torch.randn(C_, generator=g)     # norm far below the 1e-8 clamp
    f = G.bf16r(f) if dtype == "bf16" else f
    x = torch.randint(0, w, (V, N, P), generator=g)
    y = torch.randint(0, h, (V, N, P), generator=g)
    fov = torch.ones(V, N, P, dtype=torch.bool)
    fov[:, 0] = False                                     # voxel 0: every view masked -> 0 / 0 -> 0
    fov[1, 1] = False                                     # voxel 1: only view 0 in FOV (weight m_0 > m_1)
    fov[0, 2] = False                                     # voxel 2: only view 1 in FOV
    x[0, 3], y[0, 3] = 3, 2                               # voxel 3: view 0 reads the near-zero vector
    x[0, 4], y[0, 4] = -1, 5                              # voxel 4: x = -1 // 3 = -1 -> previous row's last pixel
    x[1, 5], y[1, 5] = -100, 0                            # voxel 5: in FOV, index outside the map: zero, mask counts
    x[0, 6], y[0, 6] = 1 << 31, 1                         # voxel 6: |x| > 2^30 (p1 path clamps), in FOV
    x[1, 7], y[1, 7] = -(1 << 40), -3
    pix = torch.stack([x, y], -1)
    for div in (1, 3):
        ref = lift_ref([f.double()], [div], pix, fov)
        rc, out = run_lift([f], [div], pix, fov, dtype, "f32_cl", out_cstride=C_)
        assert rc == 0
        assert torch.all(out[0] == 0)
        if div == 1 and P == 1:
            # voxel 3: the restatement's eps clamp is torch's cosine_similarity (the reference's)
            a = f[0, 2, 3].double()
            b = f[1].reshape(h * w, C_)[y[1, 3, 0] * w + x[1, 3, 0]].double()
            cos = F.cosine_similarity(a, b, 0)
            assert torch.allclose(ref[3], (cos * a + cos * b) / 2, rtol=1e-12, atol=0)
            # voxel 5: the zero feature of an in-FOV point outside the map still counts as "in view": the output is
            # 0 (cosine 0, equal masks), not half of view 0's feature
            assert torch.all(ref[5] == 0) and not torch.all(ref[4] == 0)
        check_output(out, ref, "f32_cl", C_, "edge_%s_P%d_div%d" % (dtype, P, div), dtype)


@pytest.mark.gpu
def test_lift_zero_voxels():
    from occdepth_b200 import _lib
    p = _lib.SfaParams()
    f = torch.zeros(2, 4, 4, 16, device="cuda")
    out = torch.full((4,), SENTINEL, device="cuda")
    pix = torch.zeros(2, 1, 1, 2, dtype=torch.int64, device="cuda")
    fov = torch.zeros(2, 1, 1, dtype=torch.bool, device="cuda")
    p.feat[0], p.h[0], p.w[0], p.div[0] = f.data_ptr(), 4, 4, 1
    p.n_scales, p.n_views, p.C, p.feat_dtype = 1, 2, 16, _lib.DTYPE_F32
    p.pix, p.fov, p.N, p.P = pix.data_ptr(), fov.data_ptr(), 0, 1
    p.out, p.out_mode, p.out_cstride = out.data_ptr(), _lib.SFA_OUT_F32_CL, 16
    assert _lib.lib().occd_sfa_lift_fwd(C.byref(p), _lib.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert torch.all(out.cpu() == SENTINEL)


@pytest.mark.gpu
def test_lift_index_staging_limit():
    """P x V beyond the general kernel's 200 KiB index staging is refused (OCCD_ERR_UNSUPPORTED), not overrun"""
    V, C_, P, N = 3, 32, 9, 64
    assert general_smem(V, lane_layout("f32", C_)[1], P) > 200 * 1024
    pix = torch.zeros(V, N, P, 2, dtype=torch.int64)
    fov = torch.ones(V, N, P, dtype=torch.bool)
    rc, out = run_lift([torch.randn(V, 4, 4, C_)], [1], pix, fov, "f32", "f32_cl", out_cstride=C_)
    assert rc == 3
    assert torch.all(out == SENTINEL)
