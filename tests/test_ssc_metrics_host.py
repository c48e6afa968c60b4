"""SSCMetrics on the host: argument checks of add_batch that answer before any device work, the C entry point's
refusals, and get_stats' formulas -- on hand-made confusion matrices and on the reference's results stored in
tests/golden/ssc_metrics.pt (counts from a host bincount of the same class maps)."""
import os

import numpy as np
import pytest
import torch

from occdepth_b200 import _build, _lib
from occdepth_b200.metrics import SSCMetrics, counts_from_confusion, stats_from_confusion

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ssc_metrics.pt")


def _golden():
    return torch.load(GOLDEN)


def host_confusion(pred, label, n_classes):
    """label-major confusion matrix of the voxels whose label is not 255 (np.bincount)"""
    p = pred.numpy().astype(np.int64).reshape(-1)
    g = label.numpy().astype(np.int64).reshape(-1)
    k = g != 255
    return np.bincount(g[k] * n_classes + p[k], minlength=n_classes ** 2).reshape(n_classes, n_classes)


def test_add_batch_argument_checks():
    m = SSCMetrics(20)
    p = torch.zeros(2, 4, 4, 4, dtype=torch.uint16)
    t = torch.zeros(2, 4, 4, 4, dtype=torch.float32)
    with pytest.raises(TypeError):
        m.add_batch(p.numpy(), t)
    with pytest.raises(TypeError, match="y_pred"):
        m.add_batch(p.float(), t)
    with pytest.raises(TypeError, match="y_true"):
        m.add_batch(p, t.int())
    with pytest.raises(ValueError, match="shapes"):
        m.add_batch(p, t[:, :2])
    with pytest.raises(ValueError, match="contiguous"):
        m.add_batch(p.transpose(1, 2), t.transpose(1, 2))
    with pytest.raises(ValueError, match="CUDA"):
        m.add_batch(p, t)                     # the counts are made on the device only
    with pytest.raises(ValueError, match="empty"):
        m.add_batch(p[:0], t[:0])
    assert m.counts is None                   # nothing was allocated
    for bad in (0, 65, -1):
        with pytest.raises(ValueError):
            SSCMetrics(bad)


def test_c_entry_point_refusals_without_gpu():
    _build.build()
    L = _lib.lib()
    counts = torch.zeros(401, dtype=torch.int64)
    buf = torch.zeros(64, dtype=torch.int64)
    ok = (buf.data_ptr(), _lib.DTYPE_U16, buf.data_ptr(), _lib.DTYPE_U8, 64, 20, counts.data_ptr(), None)
    for i, bad in ((0, None), (2, None), (6, None), (4, 0), (4, -5), (5, 0), (5, 65), (1, _lib.DTYPE_F32),
                   (1, _lib.DTYPE_U8), (3, _lib.DTYPE_BF16), (3, _lib.DTYPE_U16), (3, 9)):
        args = list(ok)
        args[i] = bad
        assert L.occd_ssc_confusion(*args) == _lib.ERR_ARG, (i, bad)
        assert L.occd_last_error().startswith(b"occd_ssc_confusion")
    args = list(ok)
    args[0] = buf.data_ptr() + 1                 # a uint16 map must be 2-byte aligned
    assert L.occd_ssc_confusion(*args) == _lib.ERR_ARG
    assert int(counts.abs().sum()) == 0


def test_stats_of_hand_made_counts():
    # 3 classes; rows = label, columns = prediction
    hist = np.array([[50, 3, 2],
                     [4, 10, 1],
                     [0, 2, 8]])
    tp, fp, fn, c_tp, c_fp, c_fn = counts_from_confusion(hist)
    assert tp.tolist() == [50, 10, 8] and fp.tolist() == [4, 5, 3] and fn.tolist() == [5, 5, 2]
    assert (c_tp, c_fp, c_fn) == (21, 5, 4)
    s = stats_from_confusion(hist)
    assert s["precision"] == 21 / 26 and s["recall"] == 21 / 25 and s["iou"] == 21 / 30
    want = np.array([50, 10, 8]) / (np.array([59.0, 20.0, 13.0]) + 1e-5)
    assert np.array_equal(s["iou_ssc"], want) and s["iou_ssc_mean"] == np.mean(want[1:])
    # all zero: the reference's zeros (int 0 for the completion, 0/(0 + 1e-5) per class)
    z = stats_from_confusion(np.zeros((3, 3), dtype=np.int64))
    assert (z["precision"], z["recall"], z["iou"]) == (0, 0, 0) and type(z["precision"]) is int
    assert np.array_equal(z["iou_ssc"], np.zeros(3)) and z["iou_ssc_mean"] == 0.0
    # a metric that never counted reports the same zeros; counters set by hand go through the same path
    m = SSCMetrics(3)
    assert m.get_stats()["iou_ssc_mean"] == 0.0
    m.counts = torch.tensor(hist.reshape(-1).tolist() + [0])
    assert m.get_stats()["iou"] == 21 / 30
    m.counts[-1] = 2
    with pytest.raises(ValueError, match="2 voxels"):
        m.get_stats()
    m.reset()
    assert int(m.counts.sum()) == 0


@pytest.mark.parametrize("case", ["kitti", "nyu"])
def test_formulas_equal_the_reference_results(case):
    g = _golden()[case]
    C = g["n_classes"]
    hist = host_confusion(g["pred"], g["label_i64"], C)
    assert np.array_equal(host_confusion(g["pred"], g["label_f32"], C), hist)
    assert np.array_equal(host_confusion(g["pred"], g["label_u8"], C), hist)
    tp, fp, fn, c_tp, c_fp, c_fn = counts_from_confusion(hist)
    assert np.array_equal(tp, g["tps"].numpy()) and np.array_equal(fp, g["fps"].numpy())
    assert np.array_equal(fn, g["fns"].numpy())
    assert (c_tp, c_fp, c_fn) == (g["completion_tp"], g["completion_fp"], g["completion_fn"])
    assert_stats_equal(stats_from_confusion(hist), g["stats"])
    assert (hist.sum(0) > 0).all() and (hist.sum(1) > 0).all()      # every class present
    assert int((g["label_i64"] == 255).sum()) > 0


def assert_stats_equal(got, want):
    """exact equality with the stored reference dict"""
    for k in ("precision", "recall", "iou", "iou_ssc_mean"):
        assert float(got[k]) == want[k], k
    assert np.array_equal(got["iou_ssc"], want["iou_ssc"].numpy())


@pytest.mark.reference
def test_golden_regenerates_from_the_reference():
    from oracle import gen_ssc_metrics
    new, old = gen_ssc_metrics.generate(), _golden()
    assert sorted(new) == sorted(old)
    for case in old:
        for k, v in old[case].items():
            if isinstance(v, torch.Tensor):
                assert v.dtype == new[case][k].dtype and torch.equal(v, new[case][k]), (case, k)
            elif isinstance(v, dict):
                assert_stats_equal(new[case][k], v)
            else:
                assert v == new[case][k], (case, k)
