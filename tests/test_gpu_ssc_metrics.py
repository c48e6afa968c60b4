"""SSC metrics counted on the device (occd_ssc_confusion, occdepth_b200.metrics.SSCMetrics, OccDepth's evaluation
hooks): exact counts against the reference's results (tests/golden/ssc_metrics.pt) and against torch.bincount at the
shipped grid sizes, the invalid-voxel counter, the C entry point's refusals, Lightning's test / validation hook
sequence on shipped-configuration models, the X-slab partition and the sum over ranks."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from occdepth_b200 import _lib
from occdepth_b200.metrics import SSCMetrics, counts_from_confusion, stats_from_confusion

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssc_metrics.pt")


def bincount_confusion(pred, label, C):
    """label-major confusion matrix of the voxels whose label is not 255, by torch.bincount on the device"""
    g = label.reshape(-1).to(torch.int64)
    p = pred.reshape(-1).to(torch.int64)
    k = g != 255
    return torch.bincount(g[k] * C + p[k], minlength=C * C).reshape(C, C).cpu().numpy()


def assert_stats_equal(got, want):
    for k in ("precision", "recall", "iou", "iou_ssc_mean"):
        assert float(got[k]) == float(want[k]), k
    assert np.array_equal(np.asarray(got["iou_ssc"]), np.asarray(want["iou_ssc"]))


# ---- kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["kitti", "nyu"])
@pytest.mark.parametrize("pred_dtype", [torch.uint16, torch.int64])
@pytest.mark.parametrize("label_key", ["label_f32", "label_u8", "label_i64"])
def test_counts_equal_the_reference(case, pred_dtype, label_key):
    g = torch.load(GOLDEN)[case]
    m = SSCMetrics(g["n_classes"])
    m.add_batch(g["pred"].to(pred_dtype).cuda(), g[label_key].cuda())
    hist, invalid = m.confusion()
    assert invalid == 0
    tp, fp, fn, c_tp, c_fp, c_fn = counts_from_confusion(hist)
    assert np.array_equal(tp, g["tps"].numpy()) and np.array_equal(fp, g["fps"].numpy())
    assert np.array_equal(fn, g["fns"].numpy())
    assert (c_tp, c_fp, c_fn) == (g["completion_tp"], g["completion_fp"], g["completion_fn"])
    want = dict(g["stats"])
    want["iou_ssc"] = want["iou_ssc"].numpy()
    assert_stats_equal(m.get_stats(), want)


def _maps(shape, C, skewed, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    label = torch.randint(0, C, shape, device="cuda", generator=gen)
    pred = torch.randint(0, C, shape, device="cuda", generator=gen)
    if skewed:                               # 90 % empty, mostly predicted empty
        r = torch.rand(shape, device="cuda", generator=gen)
        label[r < 0.9] = 0
        pred[(r < 0.85)] = 0
    label[torch.rand(shape, device="cuda", generator=gen) < 0.05] = 255
    return pred, label


SIZES = [("kitti", (2, 256, 256, 32), 20), ("nyu", (2, 60, 36, 60), 12)]


@pytest.mark.parametrize("name,shape,C", SIZES)
@pytest.mark.parametrize("skewed", [False, True])
def test_counts_equal_bincount_full_size(name, shape, C, skewed):
    pred, label = _maps(shape, C, skewed, seed=7)
    want = bincount_confusion(pred, label, C)
    for pdt in (torch.uint16, torch.int64):
        for ldt in (torch.float32, torch.uint8, torch.int64):
            m = SSCMetrics(C)
            m.add_batch(pred.to(pdt), label.to(ldt))
            hist, invalid = m.confusion()
            assert invalid == 0 and np.array_equal(hist, want), (pdt, ldt)
    # odd lengths and misaligned starts: the aligned vector path behind a scalar head, and the scalar path when the
    # two arrays' misalignments differ
    p16, l32 = pred.reshape(-1).to(torch.uint16), label.reshape(-1).to(torch.float32)
    n = p16.numel()
    for op, ol, ln in ((0, 0, n - 3), (1, 1, n - 8), (3, 5, n - 13), (5, 1, 7), (2, 2, 1), (0, 3, 9)):
        p, l_ = p16[op:op + ln], l32[ol:ol + ln]
        m = SSCMetrics(C)
        m.add_batch(p, l_)
        hist, invalid = m.confusion()
        assert invalid == 0 and np.array_equal(hist, bincount_confusion(p, l_, C)), (op, ol, ln)


def test_accumulates_over_batches_and_resets():
    shape, C = (1, 256, 256, 32), 20
    m = SSCMetrics(C)
    total = np.zeros((C, C), dtype=np.int64)
    for seed in range(3):
        pred, label = _maps(shape, C, skewed=seed == 1, seed=seed)
        m.add_batch(pred.to(torch.uint16), label.to(torch.float32).cpu())     # a host label is copied over
        total += bincount_confusion(pred, label, C)
    hist, invalid = m.confusion()
    assert invalid == 0 and np.array_equal(hist, total)
    assert_stats_equal(m.get_stats(), stats_from_confusion(total))
    m.reset()
    assert int(m.counts.sum()) == 0


def test_invalid_voxels_are_counted_and_refused():
    C = 20
    pred, label = _maps((1, 64, 64, 8), C, skewed=True, seed=3)
    lab = label.to(torch.float32).reshape(-1)
    prd = pred.reshape(-1).clone()             # int64 while it is edited; counted as the uint16 map
    lab[10] = 20.0                 # out of range
    lab[11] = 1.5                  # not an integer
    lab[12] = float("nan")
    lab[13] = -1.0
    lab[14] = 254.0
    lab[15], prd[15] = 3.0, 20     # prediction out of range
    lab[16], prd[16] = 255.0, 999  # ignored voxel: its prediction is not looked at
    bad = torch.zeros_like(lab, dtype=torch.bool)
    bad[10:16] = True
    m = SSCMetrics(C)
    m.add_batch(prd.to(torch.uint16), lab)
    hist, invalid = m.confusion()
    assert invalid == 6
    keep = ~bad
    assert np.array_equal(hist, bincount_confusion(prd[keep], lab[keep], C))
    with pytest.raises(ValueError, match="6 voxels"):
        m.get_stats()
    # int64 labels and predictions: negative values are invalid too
    m = SSCMetrics(C)
    m.add_batch(torch.tensor([0, -1, 5, 19], device="cuda"), torch.tensor([0, 4, -3, 19], device="cuda"))
    hist, invalid = m.confusion()
    assert invalid == 2 and hist[0, 0] == 1 and hist[19, 19] == 1 and hist.sum() == 2


def test_c_level_refusals():
    L = _lib.lib()
    counts = torch.zeros(65 * 65 + 1, dtype=torch.int64, device="cuda")
    pred = torch.zeros(1000, dtype=torch.uint16, device="cuda")
    label = torch.zeros(1000, dtype=torch.uint8, device="cuda")

    def call(pd=_lib.DTYPE_U16, ld=_lib.DTYPE_U8, n=1000, C=20):
        return L.occd_ssc_confusion(pred.data_ptr(), pd, label.data_ptr(), ld, n, C, counts.data_ptr(),
                                    _lib.stream_ptr())
    assert call(C=65) == _lib.ERR_ARG
    assert call(pd=_lib.DTYPE_F32) == _lib.ERR_ARG and call(ld=_lib.DTYPE_BF16) == _lib.ERR_ARG
    assert call(n=0) == _lib.ERR_ARG and call(n=-1) == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert int(counts.sum()) == 0                          # nothing was launched
    assert call(C=64) == 0
    torch.cuda.synchronize()
    assert int(counts[0]) == 1000 and int(counts.sum()) == 1000


# ---- model level: Lightning's test and validation loops ---------------------------------------------------------
def _case(name, **kw):
    from test_gpu_class_map import _case as case
    return case(name, **kw)


def _targets(m, batch, n, seed):
    X, Y, Z = (int(s) for s in m.full_scene_size)
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        t = torch.randint(0, m.n_classes, (1, X, Y, Z), generator=g)
        t[torch.rand(t.shape, generator=g) < 0.7] = 0
        t[torch.rand(t.shape, generator=g) < 0.1] = 255
        # the datasets' label dtypes: float32 KITTI targets, uint8 NYU targets
        out.append(t.float() if m.dataset == "kitti" else t.to(torch.uint8))
    return out


def metric_block(prefix, stats, classes):
    """the lines the reference's test_epoch_end prints (OccDepth.py:566-579)"""
    return "\n".join([
        "{}======".format(prefix),
        "Precision={:.4f}, Recall={:.4f}, IoU={:.4f}".format(stats["precision"] * 100, stats["recall"] * 100,
                                                             stats["iou"] * 100),
        "class IoU: {}, ".format(classes),
        " ".join(["{:.4f}, "] * len(classes)).format(*(stats["iou_ssc"] * 100).tolist()),
        "mIoU={:.4f}".format(stats["iou_ssc_mean"] * 100)]) + "\n"


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("name", ["kitti_b3_f32_flospdepth_2080ti", "nyu_b4_f100_2080ti"])
def test_eval_loop_shipped(name, precision, capsys, monkeypatch):
    m, batch = _case(name)
    m.set_precision(precision)
    targets = _targets(m, batch, 2, seed=11)
    C = m.n_classes
    want = np.zeros((C, C), dtype=np.int64)
    with torch.no_grad():
        y = m.predict_classes(batch)
    for t in targets:
        want += bincount_confusion(y, t.cuda(), C)
    capsys.readouterr()
    with torch.no_grad():
        for i, t in enumerate(targets):                    # trainer.test: test_step per batch, then test_epoch_end
            m.test_step(dict(batch, target=t), i)
        m.test_epoch_end([])
    out = capsys.readouterr().out
    assert out == metric_block("test", stats_from_confusion(want), m.class_names), out
    assert int(m.test_metrics.counts.sum()) == 0           # reset for the next epoch
    # trainer.validate: validation_step per batch, then validation_epoch_end's log calls for train and val
    logged = []
    monkeypatch.setattr(m, "log", lambda key, value, **kw: logged.append((key, value, kw)))
    with torch.no_grad():
        for i, t in enumerate(targets):
            m.validation_step(dict(batch, target=t), i)
        m.validation_epoch_end([])
    expect = []
    for prefix, hist in (("train", np.zeros((C, C), dtype=np.int64)), ("val", want)):
        s = stats_from_confusion(hist)
        expect += [("{}_SemIoU/{}".format(prefix, c), s["iou_ssc"][i]) for i, c in enumerate(m.class_names)]
        expect += [(prefix + "/mIoU", s["iou_ssc_mean"]), (prefix + "/IoU", s["iou"]),
                   (prefix + "/Precision", s["precision"]), (prefix + "/Recall", s["recall"])]
    assert [(k, v) for k, v, _ in logged] == expect
    assert all(kw == {"sync_dist": True} for _, _, kw in logged)
    assert int(m.val_metrics.counts.sum()) == 0


@pytest.mark.parametrize("name,world", [("kitti_b3_f32_flospdepth_2080ti", 2), ("nyu_b4_f100_2080ti", 3)])
def test_slab_counts_sum_to_the_whole(monkeypatch, name, world):
    """each rank counts its X-slab of the class map against the same planes of the target (the range its plan
    records); the sum over ranks is the unpartitioned count"""
    import gc
    from occdepth_b200.parallel import SimSlabGroup
    monkeypatch.setenv("OCCDEPTH_CUDA_GRAPH", "0")
    m, batch = _case(name)
    m.set_precision("bf16")
    target = _targets(m, batch, 1, seed=5)[0].cuda()
    whole = SSCMetrics(m.n_classes)
    with torch.no_grad():
        whole.add_batch(m.predict_classes(batch), target)
    m.invalidate_plans()
    img = batch["img"]
    B, V, _, H, W = img.shape
    pp = batch["projected_pix_%d" % m.project_scale]
    fm = batch["fov_mask_%d" % m.project_scale]
    N, P = pp[0].shape[1], pp[0].shape[2]
    grp = SimSlabGroup(world, halo=3)
    ents = []
    try:
        for r in range(world):
            m.__dict__["slab_ctx"] = grp.ctxs[r]
            with torch.no_grad():
                ents.append(m._build(B, V, H, W, N, P, img.device, batch, classes=("classes", None)))
            # the hook reads the range from the cached class-map plan
            m._class_plans().clear()
            m._class_plans()["k"] = ents[-1]
            assert m.slab_x_range() == ents[-1][0].x_range
    finally:
        m.__dict__.pop("slab_ctx", None)
        m.invalidate_plans()
    for e in ents:
        m._stage(e, batch, img, pp, fm, img.device)
    with torch.no_grad():
        SimSlabGroup.run_lockstep([e[0] for e in ents])
    ranges = [e[0].x_range for e in ents]
    assert ranges[0][0] == 0 and ranges[-1][1] == target.shape[1]
    assert all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))
    total = np.zeros((m.n_classes, m.n_classes), dtype=np.int64)
    for e, (lo, hi) in zip(ents, ranges):
        assert e[4].shape[1] == hi - lo
        part = SSCMetrics(m.n_classes)
        part.add_batch(e[4], target[:, lo:hi].contiguous())
        hist, invalid = part.confusion()
        assert invalid == 0
        total += hist
    del ents
    gc.collect()
    assert np.array_equal(total, whole.confusion()[0])
    assert_stats_equal(stats_from_confusion(total), whole.get_stats())


# ---- several ranks -----------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _shard(rank):
    g = torch.Generator().manual_seed(100 + rank)
    return torch.randint(0, 12, (1, 60, 36, 60), generator=g), torch.randint(0, 12, (1, 60, 36, 60), generator=g)


def _all_reduce_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pred, label = _shard(rank)
        m = SSCMetrics(12)
        m.add_batch(pred.to(torch.uint16).cuda(), label.to(torch.uint8))
        m.all_reduce()
        q.put((rank, m.counts.cpu().tolist()))
    finally:
        dist.destroy_process_group()


def test_all_reduce_two_processes_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_all_reduce_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = sorted(q.get(timeout=300) for _ in range(2))
    finally:
        for p in procs:
            p.join(60)
            if p.is_alive():
                p.terminate()
    assert all(p.exitcode == 0 for p in procs)
    want = np.zeros((12, 12), dtype=np.int64)
    for r in range(2):
        pred, label = _shard(r)
        k = label.reshape(-1) != 255
        want += np.bincount((label.reshape(-1)[k] * 12 + pred.reshape(-1)[k]).numpy(), minlength=144).reshape(12, 12)
    for _, counts in res:
        assert counts[:144] == want.reshape(-1).tolist() and counts[144] == 0
