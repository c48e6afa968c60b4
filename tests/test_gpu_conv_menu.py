"""The compiled convolution menu under the float64 comparator: every (precision, kernel, N tile, schedule)
instantiation, every K-chunk row width each tensor-core kernel accepts, the x-packed halo kernel's plane ring and box
mainloop, and the class map, its confidence and its probabilities on all five kernels, each launch run ALONE on
buffers filled over their whole storage and judged element by element against the float64 evaluation of its tap list
(tests/conv_replay.py), with nothing else allowed to move.

The cases (tests/conv_menu.py) reuse the shapes that steer the planner onto each menu entry (test_gpu_conv_ntiles,
test_gpu_conv_pingpong, gpu_cases) and add the epilogue variants, windows, margins, several sources, tap groups,
per-image weights and tile edges.  Equal signatures are replayed once over the module.  The last test prints what was
reached and fails on any compiled cell that no case reached."""
import time

import pytest
import torch

import conv_menu as M
import conv_replay as R
import gpu_cases as G

pytestmark = pytest.mark.gpu

_SEEN = set()
_CELLS = {}          # (precision, kernel, N tile, schedule) -> launches judged
_RB = {}             # (precision, kernel, rb) -> launches judged
_MODES = {}          # (precision, kernel, out1 mode) -> launches judged
_RING = {}           # (precision, 'ring' | 'box') -> x-packed halo launches judged
_CELL_MODES = {}     # (precision, kernel, N tile, schedule) -> set of rb / out1 mode seen, for the table
_REFUSED = {}        # (precision, name) -> planner message
_MAX = R.OBSERVED.setdefault("conv_menu", {})     # precision -> observed maxima
_RAN = {}            # (family, precision) -> (launches, judged, seconds)


def _judge(op, expect, precision, failures):
    from occdepth_b200 import _lib
    info = op.info()
    for k, v in expect.items():
        if info.get(k) != v:
            failures.append("%s: plan %r, expected %s = %r" % (op.name, info, k, v))
    sig = R.signature(op)
    if sig in _SEEN:
        return 0
    _SEEN.add(sig)
    R.fill(op, R.seed_of(sig))
    snap = R.Snapshot(op)
    op.run(_lib.stream_ptr())
    torch.cuda.synchronize()
    ref = R.reference(snap)
    fails, stats = R.check_op(op, snap, ref, info)
    kern = R.IMPL_NAME[op.impl]
    rb = info["KC"] * op.srcs[0].esize
    mode = snap.D["out1_mode"]
    cell = (precision, kern, info["N_tile"], info["schedule"])
    _CELLS[cell] = _CELLS.get(cell, 0) + 1
    _CELL_MODES.setdefault(cell, set()).update({"rb%d" % rb, "m%d" % mode})
    if kern != "simt":
        _RB[(precision, kern, rb)] = _RB.get((precision, kern, rb), 0) + 1
    _MODES[(precision, kern, mode)] = _MODES.get((precision, kern, mode), 0) + 1
    if kern == "halox":
        key = (precision, "ring" if info["ring"] else "box")
        _RING[key] = _RING.get(key, 0) + 1
    R._merge(_MAX.setdefault(precision, {}), stats)
    if fails:
        failures.append("launch on the %s kernel (%s, N tile %d, rb %d, out1 mode %d):\n    %s\n    signature: %r"
                        % (kern, info["schedule"], info["N_tile"], rb, mode, "\n    ".join(fails), dict(sig)))
    return 1


@pytest.mark.parametrize("precision", G.PRECISIONS)
@pytest.mark.parametrize("family", M.FAMILIES)
def test_menu_family(family, precision):
    t0 = time.time()
    dev = torch.device("cuda")
    failures = []
    items = M.build(family, precision, dev)
    judged = 0
    for op, expect in items:
        judged += _judge(op, expect, precision, failures)
    del items
    torch.cuda.empty_cache()
    _RAN[(family, precision)] = (len(failures), judged, time.time() - t0)
    print("\nconv menu %s [%s]: %d distinct launches judged here, %.1f s" % (family, precision, judged,
                                                                          time.time() - t0))
    assert not failures, "%d failure(s):\n%s" % (len(failures), "\n".join(failures[:8]))


@pytest.mark.parametrize("precision", G.PRECISIONS)
def test_refusals(precision):
    """per-tap class probabilities above kProbsMaxN, and per-image weights on the halo kernels"""
    dev = torch.device("cuda")
    for name, (build, exc, words) in M.refusals().items():
        with pytest.raises(exc) as e:
            build(precision, dev)
        assert words in str(e.value), (name, str(e.value))
        _REFUSED[(precision, name)] = str(e.value)


def test_coverage_and_constants():
    """after the sweep: the table instantiation x rb x mode -> launches judged; every compiled cell reached, every
    K-chunk row width on every tensor-core kernel, ring and box, modes 3 / 4 / 5 on all five kernels; the comparator's
    constants no more than twice the observed maxima.  C_ACC and A_ACT are set by the shipped sweep
    (test_gpu_conv_replay.py), whose long sums reach the larger ratios: their bound is checked over both sweeps when
    that one ran in this session too; A_SM is checked against this sweep alone."""
    if len(_RAN) != len(M.FAMILIES) * len(G.PRECISIONS):
        pytest.skip("the whole sweep did not run in this session")
    import os
    import sys
    sys.path.insert(0, os.path.join(M.ROOT, "tools"))
    import shipped_configs as sc
    gpu, power = sc.card()
    total = sum(v[2] for v in _RAN.values())
    lines = ["%-5s %-6s N %3d %-12s %4d launches  %s" % (c + (n, " ".join(sorted(_CELL_MODES[c]))))
             for c, n in sorted(_CELLS.items())]
    print("\nconv menu coverage (%s, power limit %s; %d distinct launches, %.0f s wall for the sweep):\n%s"
          % (gpu, power, len(_SEEN), total, "\n".join(lines)))
    print("rb: %s" % {"%s/%s/rb%d" % k: n for k, n in sorted(_RB.items())})
    print("out1 modes: %s" % {"%s/%s/m%d" % k: n for k, n in sorted(_MODES.items())})
    print("x-packed halo mainloop: %s" % {"%s/%s" % k: n for k, n in sorted(_RING.items())})
    print("refused: %s" % _REFUSED)
    for p in sorted(_MAX):
        print("observed maxima [%s]: %s   constants: C_ACC %.3g, A_ACT %s, A_SM %.3g"
              % (p, {k: "%.3g" % v for k, v in sorted(_MAX[p].items())}, R.C_ACC[p], R.A_ACT[p], R.A_SM[p]))
        G.record("conv_menu", p, gpu=gpu, power_limit=power, wall_s=round(total), launches=len(_SEEN), **_MAX[p])
    missing = sorted(M.compiled_cells() - set(_CELLS))
    assert not missing, "compiled instantiations no case reached: %s" % missing
    for p in G.PRECISIONS:
        for kern in M.TC_KERNELS:
            for rb in (32, 64, 128):
                assert (p, kern, rb) in _RB, "no %s launch with rb %d in %s" % (kern, rb, p)
        assert (p, "ring") in _RING and (p, "box") in _RING, (p, _RING)
        for kern in M.IMPL:
            for mode in M.MODE_NUM.values():
                assert (p, kern, mode) in _MODES, "out1 mode %d never ran on the %s kernel in %s" % (mode, kern, p)
        assert _MAX[p]["acc"] <= R.C_ACC[p] and _MAX[p]["softmax"] <= R.A_SM[p], (p, _MAX[p])
        assert R.A_SM[p] <= 2 * max(_MAX[p]["softmax"], 0.0), (p, R.A_SM[p], _MAX[p])
        shipped = R.OBSERVED.get("conv_replay", {}).get(p)
        if shipped is None:
            print("[%s] C_ACC and A_ACT: the shipped sweep did not run in this session; their bound is its test" % p)
            continue
        both = dict(_MAX[p])
        R._merge(both, shipped)
        assert R.C_ACC[p] <= 2 * both["acc"], (p, both)
        for act, a in R.A_ACT[p].items():
            assert a <= 2 * max(both.get(act, 0.0), 0.0), (p, act, a, both)
