"""Common forward plumbing of the drop-in modules: planar fp32 in/out, planned CUDA launches inside."""
import torch
import torch.nn as nn

from ..engine import CL, PRECISIONS, Plan, default_precision, require_cuda


class B200Module(nn.Module):
    """nn.Module whose forward replays a cached `Plan` built by `emit(plan, x: CL) -> CL | dict`.

    Parameters/buffers are ordinary nn.Module state (so `state_dict` matches the reference); the plan snapshots
    them (BN folded, bf16 packed) on first use and is dropped whenever a state_dict is loaded.
    Forward-only: eval() mode on a CUDA device; anything else raises (there is no CPU fallback).
    """

    def _plans(self):
        d = self.__dict__.get("_plan_cache")
        if d is None:
            d = {}
            self.__dict__["_plan_cache"] = d
        return d

    def enable_slab_parallel(self, ctx):
        """X-slab partition of one frame over the ranks of `ctx` (parallel.SlabContext): forward() then takes /
        returns this rank's X-slab of every 3-D tensor and exchanges halo planes with its neighbours."""
        self.__dict__["slab_ctx"] = ctx
        self.invalidate_plans()
        return self

    @property
    def precision(self):
        """arithmetic mode of this module's planned forward: 'tf32' (reference precision, default) or 'bf16'"""
        return self.__dict__.get("_precision") or default_precision()

    def set_precision(self, precision):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %r" % (PRECISIONS,))
        for m in self.modules():
            if isinstance(m, B200Module):
                m.__dict__["_precision"] = precision
        self.invalidate_plans()
        return self

    def param_stamp(self):
        """cheap fingerprint of the weights a plan snapshots: (storage pointer, in-place version) of every parameter
        and buffer, so load_state_dict (on this module or any child), param.copy_() and optimiser steps all rebuild
        the plan.  Writes through `param.data` bypass autograd's version counter: call invalidate_plans() after those."""
        ts = self.__dict__.get("_stamp_tensors")
        if ts is None:      # the tensor list is cached (module-tree walks cost ~1 ms for the full model); _apply and
            ts = list(self.parameters()) + list(self.buffers())     # load_state_dict drop it
            self.__dict__["_stamp_tensors"] = ts
        return hash(tuple((t.data_ptr(), t._version) for t in ts))

    def _class_plans(self):
        """plans of OccDepth.predict_classes: a cache of their own, so that forward and predict_classes on the same
        shapes keep one plan each; dropped together with _plans()"""
        return self.__dict__.setdefault("_class_plan_cache", {})

    def invalidate_plans(self):
        for m in self.modules():
            if isinstance(m, B200Module):
                m.__dict__["_plan_cache"] = {}
                m.__dict__["_class_plan_cache"] = {}

    def _load_from_state_dict(self, *a, **k):
        self.__dict__["_plan_cache"] = {}
        self.__dict__["_class_plan_cache"] = {}
        self.__dict__["_stamp_tensors"] = None
        return super()._load_from_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self.__dict__["_plan_cache"] = {}
        self.__dict__["_class_plan_cache"] = {}
        r = super()._apply(fn, *a, **k)
        self.__dict__["_stamp_tensors"] = None      # buffers are re-created by _apply
        return r

    def _check_mode(self, x):
        require_cuda(x, type(self).__name__ + ".forward")
        if self.training:
            raise RuntimeError("%s: occdepth_b200 implements the forward/inference path only; call .eval() "
                               "(BatchNorm is folded from running statistics)" % type(self).__name__)

    def _get_plan(self, x):
        """(plan, input CL, emit() result) for planar input x, built on first use"""
        self._check_mode(x)
        slab = self.__dict__.get("slab_ctx")
        key = (tuple(x.shape), str(x.device), None if slab is None else (slab.rank, slab.world), self.precision,
               self.param_stamp())
        ent = self._plans().get(key)
        if ent is None:
            self._plans().clear()      # one live plan per module: stale weight snapshots are dropped, not kept
            plan = Plan(x.device, slab=slab, precision=self.precision)
            if x.dim() == 4:
                B, C_, H, W = x.shape
                D = 1
            else:
                B, C_, D, H, W = x.shape
            xin = plan.alloc(B, D, H, W, C_)
            with torch.no_grad():
                y = self.emit(plan, xin)
            ent = (plan, xin, y)
            self._plans()[key] = ent
        return ent

    def _run_planar(self, x, squeeze_d=False):
        """x: planar fp32 [B,C,D,H,W] / [B,C,H,W]; returns emit()'s CL output(s) converted back to planar fp32."""
        with torch.cuda.device(x.device):     # kernels, tensor maps and function attributes follow the tensor
            plan, xin, y = self._get_plan(x)
            CL.from_planar(x, out=xin)
            plan.run()
            return _to_planar(y, squeeze_d)


def _to_planar(y, squeeze_d):
    if isinstance(y, CL):
        return y.to_planar(squeeze_d)
    if isinstance(y, dict):
        return {k: _to_planar(v, squeeze_d) for k, v in y.items()}
    if isinstance(y, (tuple, list)):
        return type(y)(_to_planar(v, squeeze_d) for v in y)
    return y  # already a torch tensor (fp32 planar written by a kernel)
