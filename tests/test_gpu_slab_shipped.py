"""X-slab partition of one frame for every shipped configuration (tools/shipped_configs.py, at its real shapes): the R
rank plans, built with parallel.SimSlabGroup and run in lock-step on one GPU, must reproduce the unpartitioned
forward bit for bit in both precisions -- the concatenated slabs of the logits and 3-D features, the columns of
P_logits, and every rank's whole depth_pred.  The released models also run at 4 ranks (the NYU one on uneven slabs
and CRP mega-context shards), the released KITTI model at 8, and every dataset / CRP combination at uneven world
sizes up to the largest its grid allows.  The infer_mode route (caller-supplied sampling grids, staged per window)
runs partitioned too."""
import gc
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = [("nyu_b4_f100_2080ti", 2), ("nyu_b4_f100_2080ti", 4),
         ("kitti_b3_f32_flospdepth_2080ti", 2), ("kitti_b3_f32_flospdepth_2080ti", 4),
         ("kitti_b3_f32_flospdepth_2080ti", 8),
         ("kitti_b3_f24_flospdepth_mono_2080ti", 2),
         ("kitti_b7_f64_flosp_a100", 2), ("kitti_b7_f64_flospdepth_a100", 2),
         ("nyu_b7_f200_v100", 2), ("nyu_b7_f200_v100", 4),
         # uneven slabs: KITTI with the CRP at 3 (48/40/40 planes, mega-context shards 6/5/5 padded to 6), 6 and 7
         # ranks, without it at 10; NYU at 3 and 5
         ("kitti_b3_f32_flospdepth_2080ti", 3), ("kitti_b3_f32_flospdepth_2080ti", 6),
         ("kitti_b7_f64_flosp_a100", 3), ("kitti_b7_f64_flospdepth_a100", 7),
         ("kitti_b3_f24_flospdepth_mono_2080ti", 10),
         ("nyu_b4_f100_2080ti", 3), ("nyu_b4_f100_2080ti", 5), ("nyu_b7_f200_v100", 3)]

_MODELS = {}


def _tools():
    p = os.path.join(ROOT, "tools")
    if p not in sys.path:
        sys.path.insert(0, p)
    import shipped_configs
    import slab_sim
    return shipped_configs, slab_sim


def _case(name, infer_mode=False):
    # the previous case's rank plans hold reference cycles (ops <-> plan): collect them before building more
    gc.collect()
    torch.cuda.empty_cache()
    key = (name, infer_mode)
    if key not in _MODELS:
        _MODELS.clear()
        torch.cuda.empty_cache()
        sc, _ = _tools()
        m, batch, _ = sc.make_case(name, infer_mode=infer_mode)
        batch = sc.to_cuda(batch)
        if infer_mode:
            # what a deployment supplies instead of camera matrices: one sampling grid per camera (partly outside
            # [-1, 1]) and the scaled pixel sizes
            X, Y, Z = (int(v) for v in m.flosp_depth.voxel_num.tolist())
            V = batch["img"].shape[1]
            g = torch.Generator().manual_seed(3)
            batch["grids"] = [(torch.rand(1, X, Y, Z, 3, generator=g) * 2.4 - 1.2).cuda() for _ in range(V)]
            batch["scaled_pixel_size"] = (torch.rand(V, 1, generator=g) + 0.5).cuda()
        _MODELS[key] = (m.cuda(), batch)
    return _MODELS[key]


def _compare(ref, outs):
    keys = set(ref)
    assert all(set(o) == keys for o in outs)
    for k in sorted(keys):
        if k == "depth_pred":
            for r, o in enumerate(outs):
                assert _bits_equal(o[k], ref[k]), (k, r)
            continue
        got = torch.cat([o[k] for o in outs], 3 if k == "P_logits" else 2)
        assert _bits_equal(got, ref[k]), (k, float((got - ref[k]).abs().max()) if got.shape == ref[k].shape
                                          else (tuple(got.shape), tuple(ref[k].shape)))


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name,world", CASES)
def test_slab_matches_unpartitioned_bit_for_bit(monkeypatch, name, world, precision):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    _, slab_sim = _tools()
    m, batch = _case(name)
    m.set_precision(precision)
    with torch.no_grad():
        ref = m(batch)
    m.invalidate_plans()
    grp, ents = slab_sim.rank_plans(m, batch, world)
    outs = slab_sim.run_lockstep(m, ents, batch)
    del ents
    assert grp.ctxs[0].n_exchanges > 0
    assert {"ssc_logit", "x3d_l1", "x3d_l2", "x3d_l3"} <= set(ref)
    _compare(ref, outs)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("world", [2, 3])
def test_infer_mode_slab_matches_unpartitioned_bit_for_bit(monkeypatch, world, precision):
    """released KITTI model built for infer_mode (no CRP: 32 units of 4 planes, 64/64 or 44/44/40): each rank stages
    only its window's rows of the caller's grids and samples them at their whole-grid index"""
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    _, slab_sim = _tools()
    m, batch = _case("kitti_b3_f32_flospdepth_2080ti", infer_mode=True)
    m.set_precision(precision)
    with torch.no_grad():
        ref = m(batch)
    m.invalidate_plans()
    grp, ents = slab_sim.rank_plans(m, batch, world)
    assert [e[0].flosp_state["window"] for e in ents] == [(lo, hi - lo) for lo, hi in grp.ctxs[0].bounds]
    outs = slab_sim.run_lockstep(m, ents, batch)
    del ents
    assert "ssc_logit" in ref and "depth_pred" in ref
    _compare(ref, outs)
