"""Per-launch convolution parity at the shipped geometries: every distinct convolution the six shipped configurations
plan (tools/shipped_configs.py, real shapes; forward plan, predict_classes plan, and one X-slab rank plan each for the
released KITTI model at 4 ranks and the NYU B7 model at 3) is run ALONE, in place, in its real buffers with its real
descriptor, and compared element by element with the float64 evaluation of its tap list (tests/conv_replay.py).

Every buffer a launch reaches is filled over its whole storage first -- margin planes, channels outside the windows,
residuals, run-time weights, and the outputs -- so a missed store shows and "nothing else moves" is a real check.  Two
launches with equal signatures (same descriptor numbers, same kernel, tile box, N tile, K chunk, stages, grid and
schedule) are the same launch on different data: only the first is replayed, over the whole module.  Nothing is timed
and no launch is repeated."""
import contextlib
import gc
import io
import os
import sys
import time

import pytest
import torch

import conv_replay as R
import gpu_cases as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti", "kitti_b3_f24_flospdepth_mono_2080ti",
         "kitti_b7_f64_flosp_a100", "kitti_b7_f64_flospdepth_a100", "nyu_b7_f200_v100"]
# (world, rank) of the slab rank plan replayed as well: uneven slabs, margin planes, a CRP mega-context shard
SLAB = {"kitti_b3_f32_flospdepth_2080ti": (4, 1), "nyu_b7_f200_v100": (3, 1)}

_MODEL = {}
_SEEN = set()
_COVER = {}          # (kernel, schedule, N tile, rb) -> launches replayed
_CLASS_MAP = set()   # (kernel, out1 mode) of every class-map epilogue that ran
_MAX = R.OBSERVED.setdefault("conv_replay", {})   # precision -> observed maxima (conv_replay.check, check_prob)
_RAN = {}            # (name, precision) -> (launches, replayed, seconds)


def _tools():
    p = os.path.join(ROOT, "tools")
    if p not in sys.path:
        sys.path.insert(0, p)
    import shipped_configs
    import slab_sim
    return shipped_configs, slab_sim


def _case(name):
    if name not in _MODEL:
        _MODEL.clear()
        gc.collect()
        torch.cuda.empty_cache()
        sc, _ = _tools()
        m, batch, _ = sc.make_case(name)
        _MODEL[name] = (m.cuda(), sc.to_cuda(batch))
    return _MODEL[name]


def _build(m, batch, classes=None, slab=None):
    _, slab_sim = _tools()
    B, V, H, W, N, P, dev = slab_sim._shape_args(m, batch)
    if slab is not None:
        m.__dict__["slab_ctx"] = slab
    try:
        with torch.no_grad(), torch.cuda.device(dev), contextlib.redirect_stdout(io.StringIO()):
            return m._build(B, V, H, W, N, P, dev, batch, classes=classes)[0]
    finally:
        m.__dict__.pop("slab_ctx", None)


def _replay(plan, what, precision, failures, count):
    from occdepth_b200 import _lib
    from occdepth_b200.engine import ConvOp
    st = _lib.stream_ptr()
    for op in plan.ops:
        if not isinstance(op, ConvOp):
            continue
        count[0] += 1
        sig = R.signature(op)
        if sig in _SEEN:
            continue
        _SEEN.add(sig)
        count[1] += 1
        info = op.info()
        R.fill(op, R.seed_of(sig))
        snap = R.Snapshot(op)
        op.run(st)
        torch.cuda.synchronize()
        ref = R.reference(snap)
        fails, stats = R.check_op(op, snap, ref, info)
        kernel = R.IMPL_NAME[op.impl]
        key = (kernel, info["schedule"], info["N_tile"], info["KC"] * op.srcs[0].esize)
        _COVER[key] = _COVER.get(key, 0) + 1
        if snap.D["out1_mode"] in R.CLASS_OUT1:
            _CLASS_MAP.add((kernel, snap.D["out1_mode"]))
        R._merge(_MAX.setdefault(precision, {}), stats)
        if fails:
            failures.append("%s, launch %r on the %s kernel (%s schedule):\n    %s\n    signature: %r"
                            % (what, op.name, kernel, info["schedule"], "\n    ".join(fails), dict(sig)))
        del snap, ref


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_every_planned_convolution_alone(monkeypatch, name, precision):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    from occdepth_b200.parallel import SimSlabGroup
    t0 = time.time()
    m, batch = _case(name)
    m.set_precision(precision)
    m.invalidate_plans()
    failures, count = [], [0, 0]
    # the class-map plan of every other configuration remaps its labels
    lut = tuple((7 * i + 3) % 251 for i in range(m.n_classes)) if NAMES.index(name) % 2 else None
    # the confidence and probability plans add only their classifier launch: the others deduplicate by signature
    variants = [("forward", dict()), ("predict_classes", dict(classes=("classes", lut))),
                ("predict_classes(confidence=True)", dict(classes=m._class_key(lut, confidence=True))),
                ("predict_classes(probabilities=True)", dict(classes=m._class_key(lut, probabilities=True)))]
    if name in SLAB:
        world, rank = SLAB[name]
        variants.append(("slab rank %d of %d" % (rank, world), dict(slab=SimSlabGroup(world, halo=3).ctxs[rank])))
    for what, kw in variants:
        plan = _build(m, batch, **kw)
        _replay(plan, "%s [%s] %s plan" % (name, precision, what), precision, failures, count)
        del plan
        gc.collect()                # plans hold reference cycles (ops <-> plan): free their buffers now
        torch.cuda.empty_cache()
    _RAN[(name, precision)] = (count[0], count[1], time.time() - t0)
    print("\nconv replay %s [%s]: %d conv launches planned, %d distinct signatures replayed here, %.0f s"
          % (name, precision, count[0], count[1], _RAN[(name, precision)][2]))
    assert count[1] > 0 or len(_SEEN) > 0
    assert not failures, "%d launch(es) failed:\n%s" % (len(failures), "\n".join(failures[:8]))


def test_coverage_and_constants():
    """after the sweep: which (kernel, schedule, N tile, K-chunk row bytes) it reached, the observed maxima, and that
    the comparator's constants are no more than twice those maxima"""
    if len(_RAN) != 2 * len(NAMES):
        pytest.skip("the whole sweep did not run in this session")
    sc, _ = _tools()
    gpu, power = sc.card()
    lines = ["%-6s %-12s N tile %3d  rb %3d: %4d launches" % (k + (n,)) for k, n in sorted(_COVER.items())]
    total = sum(v[2] for v in _RAN.values())
    print("\nconv replay coverage (%s, power limit %s; %d distinct launches, %.0f s wall for the sweep):\n%s"
          % (gpu, power, len(_SEEN), total, "\n".join(lines)))
    print("class-map epilogue (kernel, out1 mode) on: %s" % sorted(_CLASS_MAP))
    for p in sorted(_MAX):
        print("observed maxima [%s] (acc per sqrt(K) S): %s   constants: C_ACC %.3g, A_ACT %s, A_SM %.3g"
              % (p, {k: "%.3g" % v for k, v in sorted(_MAX[p].items())}, R.C_ACC[p], R.A_ACT[p], R.A_SM[p]))
        G.record("conv_replay", p, gpu=gpu, power_limit=power, wall_s=round(total), launches=len(_SEEN),
                 coverage=["%s/%s/N%d/rb%d" % k for k in sorted(_COVER)], **_MAX[p])
    kernels = {k[0] for k in _COVER}
    assert {"tc", "tcx", "halo", "halox"} <= kernels, kernels
    assert {"cooperative", "pingpong"} <= {k[1] for k in _COVER}
    assert {m for _, m in _CLASS_MAP} == set(R.CLASS_OUT1), _CLASS_MAP
    for p in ("tf32", "bf16"):
        assert R.C_ACC[p] <= 2 * _MAX[p]["acc"], (p, _MAX[p])
        for act, a in R.A_ACT[p].items():
            assert a <= 2 * max(_MAX[p].get(act, 0.0), 0.0), (p, act, a, _MAX[p])
        assert R.A_SM[p] <= 2 * max(_MAX[p]["softmax"], 0.0), (p, R.A_SM[p], _MAX[p])
