"""Per-launch parity of the non-convolution launches at the shipped geometries: every distinct helper launch that the
six shipped configurations plan (tools/shipped_configs.py; forward and predict_classes plans, one X-slab rank plan
each for KITTI B3 at 4 ranks and NYU B7 at 3, FlospDepth's infer_mode grids route, NYU's two-frame depth_items
route) is recorded from the plan itself (tests/launch_replay.py), run ALONE in its real buffers after the plan ran
once on the case's batch -- so its inputs are the model's real intermediates -- and compared with its float64
reference.

Before each launch the declared output regions and the channels outside each channels-last input window are
poisoned with NaN; afterwards every output is checked, every other byte of every storage it reaches must hold what it
held before, and the plan's data is put back.  Equal signatures are the same launch on different data: only the
first is replayed, over the whole module.  Nothing is timed and no launch is repeated."""
import contextlib
import gc
import io
import os
import sys
import time

import pytest
import torch

import gpu_cases as G
import launch_replay as LR

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["nyu_b4_f100_2080ti", "kitti_b3_f32_flospdepth_2080ti", "kitti_b3_f24_flospdepth_mono_2080ti",
         "kitti_b7_f64_flosp_a100", "kitti_b7_f64_flospdepth_a100", "nyu_b7_f200_v100"]
SLAB = {"kitti_b3_f32_flospdepth_2080ti": (4, 1), "nyu_b7_f200_v100": (3, 1)}
INFER = "kitti_b3_f24_flospdepth_mono_2080ti"
FRAMES = "nyu_b4_f100_2080ti"

_SEEN = set()
_NAMES = {}          # entry point -> launches replayed
_MENU = {}           # menus reached: ("dw", K, stride) -> {(cvb, TH, PX)}, ("lift",) -> {(dtype, V, NV, G)}
_MAX = {}            # precision -> observed maxima
_RAN = {}


def _tools():
    p = os.path.join(ROOT, "tools")
    if p not in sys.path:
        sys.path.insert(0, p)
    import shipped_configs
    import slab_sim
    return shipped_configs, slab_sim


def _replay(recs, st, what, precision, failures, count):
    from occdepth_b200 import _lib
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = _lib.stream_ptr()
    for rec in recs:
        count[0] += 1
        sig = LR.signature(rec, st)
        if sig in _SEEN:
            continue
        _SEEN.add(sig)
        count[1] += 1
        fails, stats, L = LR.replay(rec, st, stream)
        _NAMES[rec[0]] = _NAMES.get(rec[0], 0) + 1
        if rec[0] == "occd_dwconv2d_tiled_fwd":
            _MENU.setdefault(("dw", L.a["K"], L.a["stride"]), set()).add(LR.dw_menu(L.a, n_sms))
        if rec[0] == "occd_sfa_lift_fwd":
            _MENU.setdefault(("lift",), set()).add(LR.lift_menu(L.a["p"]))
        LR.CR._merge(_MAX.setdefault(precision, {}), stats)
        if fails:
            failures.append("%s, %s:\n    %s\n    signature: %r" % (what, rec[0], "\n    ".join(fails), sig))
        del L


def _plans(name, precision):
    """-> [(what, records, storages)] of the case's plans, each run once on the batch before it is recorded"""
    sc, slab_sim = _tools()
    out = []
    m, batch, _ = sc.make_case(name)
    m = m.cuda()
    batch = sc.to_cuda(batch)
    m.set_precision(precision)
    lut = tuple((7 * i + 3) % 251 for i in range(m.n_classes)) if NAMES.index(name) % 2 else None
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        for what, run, cache in (("forward", lambda: m(batch), m._plans),
                                 ("predict_classes", lambda: m.predict_classes(batch, inv_map=lut), m._class_plans)):
            m.invalidate_plans()
            with LR.Recording() as R:
                run()
                torch.cuda.synchronize()
                ent = list(cache().values())[0]
                out.append((what, R.calls(ent[0]), LR.Storages(LR.plan_tensors(ent[0], ent[1:]))))
                state = getattr(ent[0], "flosp_state", None)
                sps = None if state is None else state["sps"].clone()
        m.invalidate_plans()
        if name in SLAB:
            world, rank = SLAB[name]
            with LR.Recording() as R:
                _, ents = slab_sim.rank_plans(m, batch, world)
                slab_sim.run_lockstep(m, ents, batch)
                out.append(("slab rank %d of %d" % (rank, world), R.calls(ents[rank][0]),
                            LR.Storages(LR.plan_tensors(ents[rank][0], ents[rank][1:]))))
            del ents
        if name == FRAMES:
            from camera_frames import nyu_frame
            frames = []
            for i in range(2):
                f = nyu_frame(1 + i)
                f["img_hw"] = sc.NYU_IMG
                frames.append(f)
            m.invalidate_plans()
            with LR.Recording() as R:
                m.predict_frames(frames)
                torch.cuda.synchronize()
                ent = list(m._class_plans().values())[0]
                out.append(("predict_frames x2", R.calls(ent[0]), LR.Storages(LR.plan_tensors(ent[0], ent[1:]))))
    if name == INFER:
        # the deployment route's grids: the frustum grids of the forward plan's own camera tables
        rec, st = next((r, s) for _, rs, s in out for r in rs if r[0] == "occd_frustum_sample_window_fwd")
        a = LR.named(rec)
        cams = LR.flat(st, a["cams"], a["V"] * 40, torch.float32).view(st.by_key)
        mi, bi, _ = sc.make_case(name, infer_mode=True)
        mi = mi.cuda()
        bi = sc.to_cuda(bi)
        bi["grids"] = [LR.frustum_grid_f64(*LR._cams_of(cams[v * 40:(v + 1) * 40]), (a["X"], a["Y"], a["Z"]),
                                           (a["img_h"], a["img_w"]), a["Dn"], a["dmin"], a["dmax"]).float()
                       for v in range(a["V"])]
        bi["scaled_pixel_size"] = sps
        mi.set_precision(precision)
        with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()), LR.Recording() as R:
            mi(bi)
            torch.cuda.synchronize()
            ent = list(mi._plans().values())[0]
            out.append(("infer_mode forward", R.calls(ent[0]), LR.Storages(LR.plan_tensors(ent[0], ent[1:]))))
    return out


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_every_planned_helper_launch_alone(monkeypatch, name, precision):
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    t0 = time.time()
    failures, count = [], [0, 0]
    for what, recs, st in _plans(name, precision):
        _replay(recs, st, "%s [%s] %s plan" % (name, precision, what), precision, failures, count)
        del recs, st
    gc.collect()
    torch.cuda.empty_cache()
    _RAN[(name, precision)] = (count[0], count[1], time.time() - t0)
    print("\nlaunch replay %s [%s]: %d helper launches recorded, %d distinct signatures replayed here, %.0f s"
          % (name, precision, count[0], count[1], _RAN[(name, precision)][2]))
    assert count[0] > 0
    assert not failures, "%d launch(es) failed:\n%s" % (len(failures), "\n".join(failures[:8]))


def test_coverage_and_constants():
    if len(_RAN) != 2 * len(NAMES):
        pytest.skip("the whole sweep did not run in this session")
    sc, _ = _tools()
    gpu, power = sc.card()
    total = sum(v[2] for v in _RAN.values())
    print("\nlaunch replay coverage (%s, power limit %s; %d distinct launches, %.0f s wall):" % (gpu, power, len(_SEEN),
                                                                                               total))
    for n, k in sorted(_NAMES.items()):
        print("  %-36s %4d" % (n, k))
    for k, v in sorted(_MENU.items(), key=str):
        print("  menu %s: %s" % (k, sorted(v, key=str)))
    for p in sorted(_MAX):
        print("observed maxima [%s]: %s" % (p, {k: "%.3g" % v for k, v in sorted(_MAX[p].items())}))
        print("constants      [%s]: %s" % (p, {f: "%.3g" % c[p] for f, c in sorted(LR.C_ACC.items())}))
        G.record("launch_replay", p, gpu=gpu, power_limit=power, wall_s=round(total), launches=len(_SEEN),
                 entry_points=sorted(_NAMES), **_MAX[p])
    assert set(_NAMES) == set(LR.SPECS), set(LR.SPECS) - set(_NAMES)
    for p in ("tf32", "bf16"):
        for fam, c in LR.C_ACC.items():
            if fam in _MAX[p]:
                assert c[p] <= 2 * max(_MAX[p][fam], 0.0), (p, fam, c[p], _MAX[p][fam])
        for act, a in LR.A_ACT[p].items():
            assert a <= 2 * max(_MAX[p].get("dw." + act, 0.0), 0.0), (p, act, a, _MAX[p])
