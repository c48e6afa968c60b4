"""Generates tests/golden/ssc_metrics.pt by running the UNMODIFIED reference SSCMetrics (loss/sscMetrics.py) on
seeded class maps and labels:  OCCDEPTH_REFERENCE=<checkout of the original project> python -m oracle.gen_ssc_metrics

Two cases, a small KITTI-like grid (20 classes) and a small NYU-like one (12 classes), each a batch of 2 with 255
(ignore) labels, a dominant empty class and every class present among labels and predictions.  The fixture holds the
class map (uint16), the labels in the three dtypes the datasets produce (float32 KITTI, uint8 NYU, int64 torch), and
the reference's accumulators (tps, fps, fns, completion tp / fp / fn) and get_stats() dict after add_batch.
"""
import os
import sys
import types

import numpy as np
import torch

from . import ref_import

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ssc_metrics.pt")

CASES = {"kitti": ((2, 32, 32, 4), 20, 0), "nyu": ((2, 15, 9, 15), 12, 1)}    # shape, classes, seed


def case_inputs(shape, n_classes, seed):
    """(pred uint16, label int64) with ~60 % empty labels, ~10 % 255, predictions right ~half of the time"""
    rng = np.random.default_rng(seed)
    label = rng.integers(1, n_classes, size=shape)
    label[rng.random(shape) < 0.6] = 0
    label[rng.random(shape) < 0.1] = 255
    pred = rng.integers(0, n_classes, size=shape)
    keep = (rng.random(shape) < 0.5) & (label != 255)
    pred[keep] = label[keep]
    flat_l, flat_p = label.reshape(-1), pred.reshape(-1)
    flat_l[:n_classes] = np.arange(n_classes)            # every class present in both
    flat_p[:n_classes] = np.arange(n_classes)[::-1]
    return torch.from_numpy(pred.astype(np.uint16)), torch.from_numpy(label.astype(np.int64))


def _reference_metrics():
    """the reference's SSCMetrics class; its module imports scikit-learn for functions SSCMetrics never calls, so a
    stand-in module is installed when scikit-learn is missing"""
    ref_import._install()
    try:
        import sklearn.metrics  # noqa: F401
    except ImportError:
        sk = types.ModuleType("sklearn")
        skm = types.ModuleType("sklearn.metrics")

        def unused(*a, **k):
            raise NotImplementedError("scikit-learn stand-in")
        skm.accuracy_score = skm.precision_recall_fscore_support = unused
        sk.metrics = skm
        sys.modules.setdefault("sklearn", sk)
        sys.modules.setdefault("sklearn.metrics", skm)
    from occdepth.loss.sscMetrics import SSCMetrics
    return SSCMetrics


def generate():
    SSCMetrics = _reference_metrics()
    out = {}
    for name, (shape, n_classes, seed) in CASES.items():
        pred, label = case_inputs(shape, n_classes, seed)
        y_pred = pred.numpy().astype(np.int64)                 # np.argmax's dtype, as OccDepth.step passes it
        res = None
        for dt in (np.float32, np.uint8, np.int64):            # every label dtype gives the same counts
            m = SSCMetrics(n_classes)
            m.add_batch(y_pred, label.numpy().astype(dt))
            st = m.get_stats()
            r = dict(tps=torch.from_numpy(m.tps.copy()), fps=torch.from_numpy(m.fps.copy()),
                     fns=torch.from_numpy(m.fns.copy()), completion_tp=int(m.completion_tp),
                     completion_fp=int(m.completion_fp), completion_fn=int(m.completion_fn),
                     stats={"precision": float(st["precision"]), "recall": float(st["recall"]), "iou": float(st["iou"]),
                            "iou_ssc": torch.from_numpy(np.asarray(st["iou_ssc"], dtype=np.float64)),
                            "iou_ssc_mean": float(st["iou_ssc_mean"])})
            if res is None:
                res = r
            else:
                assert all(torch.equal(res[k], r[k]) for k in ("tps", "fps", "fns")), name
                assert res["stats"]["iou_ssc_mean"] == r["stats"]["iou_ssc_mean"], name
        out[name] = dict(n_classes=n_classes, pred=pred, label_f32=label.float(), label_u8=label.to(torch.uint8),
                         label_i64=label, **res)
    return out


def main():
    torch.save(generate(), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
