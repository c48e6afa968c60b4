"""Drop-in for the reference `occdepth/models/CRP3D.py`: CPMegaVoxels (:9-97), the 3D Context Relation Prior.

ASPP -> stride-2 mega-context conv -> n_relations 1x1x1 relation convs (sigmoid fused, raw logits written
straight into P_logits) -> the torch.bmm as wgmma GEMMs whose "weights" are the transposed mega-context
-> concat buffer written in place -> 1x1x1 resize -> Process.
"""
import torch
import torch.nn as nn

from .. import _lib
from ..engine import CL, ConvOp, FnOp, fold_bn, out_size, _round_up
from ._base import B200Module
from .modules import ASPP, Process


class CPMegaVoxels(B200Module):
    def __init__(self, feature, size, n_relations=4, bn_momentum=0.0003):
        super().__init__()
        self.size = size
        self.n_relations = n_relations
        print("n_relations", self.n_relations)
        self.flatten_size = size[0] * size[1] * size[2]
        self.feature = feature
        self.context_feature = feature * 2
        self.flatten_context_size = (size[0] // 2) * (size[1] // 2) * (size[2] // 2)
        padding = ((size[0] + 1) % 2, (size[1] + 1) % 2, (size[2] + 1) % 2)
        self.mega_context = nn.Sequential(
            nn.Conv3d(feature, self.context_feature, stride=2, padding=padding, kernel_size=3))
        self.context_prior_logits = nn.ModuleList(
            [nn.Sequential(nn.Conv3d(self.feature, self.flatten_context_size, padding=0, kernel_size=1))
             for i in range(n_relations)])
        self.aspp = ASPP(feature, [1, 2, 3])
        self.resize = nn.Sequential(
            nn.Conv3d(self.context_feature * self.n_relations + feature, feature, kernel_size=1, padding=0,
                      bias=False),
            Process(feature, nn.BatchNorm3d, bn_momentum, dilations=[1]))

    def emit(self, plan, x):
        """x: CL [B, X, Y, Z, feature] -> {"P_logits": fp32 [B, R, M, N], "x": CL}"""
        L = _lib.lib()
        B, D, H, W = x.dims
        N, M, R = self.flatten_size, self.flatten_context_size, self.n_relations
        F1, F2 = self.feature, self.context_feature
        slab = plan.slab
        conv = self.mega_context[0]
        shards = None
        if slab is None:
            assert D * H * W == N
        else:   # X-slab partition: this rank holds D of the X planes; the mega-context is all-gathered
            # each rank's X planes here and its mega-context planes (the stride-2 outputs anchored on its planes)
            lb = slab.level_bounds(self.size[0]) or [(r * D, (r + 1) * D) for r in range(slab.world)]
            n_out = out_size(self.size[0], 3, 2, conv.padding[0], 1)
            shards = [(n_out if r == slab.world - 1 else hi // 2) - lo // 2 for r, (lo, hi) in enumerate(lb)]
            assert B == 1 and sum(hi - lo for lo, hi in lb) * H * W == N and lb[slab.rank][1] - lb[slab.rank][0] == D
            N = D * H * W
        x_agg = self.aspp.emit(plan, x)
        w, b = fold_bn(conv.weight, conv.bias, None)
        F2p = _round_up(F2, 16)
        Kp = plan.kpad_for(M)
        wbuf = torch.zeros(B, 1, F2p, Kp, dtype=plan.dtype, device=plan.device)
        if shards is not None and min(shards) != max(shards):
            # uneven shards: every rank gathers max(shards) planes (its own, zero-padded), and the bmm operand is
            # transposed shard by shard, so the padding never reaches it
            cd = max(shards)
            ch, cw = (out_size(e, 3, 2, p, 1) for e, p in zip((H, W), conv.padding[1:]))
            own = CL.alloc(1, cd, ch, cw, F2, plan.device, precision=plan.precision)
            ctx = plan.conv(x_agg, w, b, stride=2, padding=conv.padding, name="crp.mega_context",
                            out=CL(own.buf[:, :shards[slab.rank]], F2))
            full = CL.alloc(1, cd * slab.world, ch, cw, F2, plan.device, precision=plan.precision)
            plan.add(slab.all_gather_op(own.buf, full.buf))
            m0, plane = 0, ch * cw
            for r, n_r in enumerate(shards):
                src = full.ptr + full.esize * r * cd * full.plane_elems
                dst = wbuf.data_ptr() + wbuf.element_size() * m0
                plan.add(FnOp(lambda st, src=src, dst=dst, P=n_r * plane: L.occd_cl_transpose(
                    src, dst, plan.lib_dtype, B, P, F2, full.cstride, 0, Kp, F2p * Kp, st), "occd_cl_transpose",
                    keep=(full, wbuf)))
                m0 += n_r * plane
            assert m0 == M
        else:
            ctx = plan.conv(x_agg, w, b, stride=2, padding=conv.padding, name="crp.mega_context")   # [B, M pos, F2]
            if slab is not None:
                _, cd, ch, cw = ctx.dims
                full = CL.alloc(1, cd * slab.world, ch, cw, F2, plan.device, precision=plan.precision)
                plan.add(slab.all_gather_op(ctx.interior(), full.buf))
                ctx = full
            assert ctx.spatial() == M
            # mega-context as the K-major B operand of the bmm: wbuf[b][f][m] = ctx[b][m][f]
            plan.add(FnOp(lambda st: L.occd_cl_transpose(ctx.ptr, wbuf.data_ptr(), plan.lib_dtype, B, M, F2,
                                                         ctx.cstride, ctx.coff, Kp, F2p * Kp, st), "occd_cl_transpose",
                          keep=(ctx, wbuf)))
        P_logits = torch.empty(B, R, M, N, dtype=torch.float32, device=plan.device)
        p_view = P_logits.view(B, R * M, D, H, W)
        cat = plan.alloc(B, D, H, W, F1 + R * F2)
        plan.add(FnOp(lambda st: L.occd_copy_channels(x.ptr, cat.ptr, plan.lib_dtype, B * N, F1, x.cstride, x.coff,
                                                      cat.cstride, cat.coff, st), "occd_copy_channels",
                      keep=(x, cat)))
        zero_bias = torch.zeros(F2, device=plan.device)
        for r in range(R):
            c = self.context_prior_logits[r][0]
            w, b = fold_bn(c.weight, c.bias, None)
            sig = plan.conv(x_agg, w, b, act="sigmoid", out1=p_view, out1_mode="planar", out1_coff=r * M,
                            name="crp.rel%d" % r)                                   # [B, N pos, M] sigmoid
            for bi in range(B):
                src = type(sig)(sig.buf[bi:bi + 1], sig.C, sig.coff, sig.d0, sig.dlen)
                dst = type(cat)(cat.buf[bi:bi + 1], F2, F1 + r * F2, cat.d0, cat.dlen)
                plan.add(ConvOp([src], [(0, 0, 0, 0)], None, zero_bias, (D, H, W), out0=dst, weight_buf=wbuf[bi],
                                name="crp.bmm%d" % r))
        conv = self.resize[0]
        w, b = fold_bn(conv.weight, conv.bias, None)
        y = plan.conv(cat, w, b, name="crp.resize")
        y = self.resize[1].emit(plan, y)
        return {"P_logits": P_logits, "x": y}

    def forward(self, input):
        return self._run_planar(input)
