"""Semantic scene completion metrics counted on the device: the drop-in for the reference's `SSCMetrics`
(loss/sscMetrics.py:40-129) as OccDepth uses it (`add_batch(y_pred, y_true)`, `get_stats()`, `reset()`).

The reference copies the logits to the host, takes np.argmax and makes three np.where passes per class.  Here
`add_batch` launches one kernel (occd_ssc_confusion) that reads the class map and the labels once and accumulates
their confusion matrix on the device, without synchronising; `get_stats` reads the matrix back once and derives the
reference's counts and its float64 formulas from it, so the statistics are identical to the reference's.
"""
import numpy as np
import torch

from . import _lib

MAX_CLASSES = 64
IGNORE_LABEL = 255
_PRED_DTYPES = {torch.uint16: _lib.DTYPE_U16, torch.int64: _lib.DTYPE_I64}
_LABEL_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.uint8: _lib.DTYPE_U8, torch.int64: _lib.DTYPE_I64}


class SSCMetrics:
    """Counters of one evaluation split.  The int64 counters ([n_classes^2 + 1]: the confusion matrix, label-major,
    then the invalid-voxel count) are created on the device of the first `add_batch`: a model is built on the CPU
    and moved afterwards, so the constructor allocates nothing."""

    def __init__(self, n_classes):
        n_classes = int(n_classes)
        if not 0 < n_classes <= MAX_CLASSES:
            raise ValueError("SSCMetrics: n_classes must be in [1, %d], got %d" % (MAX_CLASSES, n_classes))
        self.n_classes = n_classes
        self.counts = None

    def reset(self):
        if self.counts is not None:
            self.counts.zero_()

    def add_batch(self, y_pred, y_true):
        """count one batch: y_pred the class map (uint16, as predict_classes / class_map return it, or int64, a torch
        argmax) on a CUDA device; y_true the labels of the same shape (float32, uint8 or int64; 255 = ignore), on the
        same device or on the host (then copied over).  Both contiguous.  Enqueued on the current stream."""
        if not isinstance(y_pred, torch.Tensor) or not isinstance(y_true, torch.Tensor):
            raise TypeError("SSCMetrics.add_batch: y_pred and y_true must be torch tensors")
        if y_pred.dtype not in _PRED_DTYPES:
            raise TypeError("SSCMetrics.add_batch: y_pred must be uint16 or int64, got %s" % y_pred.dtype)
        if y_true.dtype not in _LABEL_DTYPES:
            raise TypeError("SSCMetrics.add_batch: y_true must be float32, uint8 or int64, got %s" % y_true.dtype)
        if tuple(y_pred.shape) != tuple(y_true.shape):
            raise ValueError("SSCMetrics.add_batch: shapes differ: %s vs %s" % (tuple(y_pred.shape), tuple(y_true.shape)))
        if y_pred.numel() == 0:
            raise ValueError("SSCMetrics.add_batch: empty batch")
        if not (y_pred.is_contiguous() and y_true.is_contiguous()):
            raise ValueError("SSCMetrics.add_batch: y_pred and y_true must be contiguous")
        if not y_pred.is_cuda:
            raise ValueError("SSCMetrics.add_batch: y_pred must be on a CUDA device (the counts are made there)")
        dev = y_pred.device
        if y_true.device != dev:
            if y_true.is_cuda:
                raise ValueError("SSCMetrics.add_batch: y_pred on %s, y_true on %s" % (dev, y_true.device))
            y_true = y_true.to(dev, non_blocking=True)
        if self.counts is not None and self.counts.device != dev:
            raise ValueError("SSCMetrics.add_batch: counting on %s, batch on %s" % (self.counts.device, dev))
        with torch.cuda.device(dev):
            if self.counts is None:
                self.counts = torch.zeros(self.n_classes ** 2 + 1, dtype=torch.int64, device=dev)
            _lib.check(_lib.lib().occd_ssc_confusion(y_pred.data_ptr(), _PRED_DTYPES[y_pred.dtype], y_true.data_ptr(),
                                                     _LABEL_DTYPES[y_true.dtype], y_pred.numel(), self.n_classes,
                                                     self.counts.data_ptr(), _lib.stream_ptr()),
                       "occd_ssc_confusion")

    def all_reduce(self, group=None):
        """sum the counters over the ranks of `group` (default: the default process group), so that every rank's
        statistics cover the whole split.  A rank that counted nothing takes part with zeros."""
        import torch.distributed as dist
        if self.counts is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
            self.counts = torch.zeros(self.n_classes ** 2 + 1, dtype=torch.int64, device=dev)
        dist.all_reduce(self.counts, op=dist.ReduceOp.SUM, group=group)

    def confusion(self):
        """(int64 numpy [n_classes, n_classes] confusion matrix, rows = label, columns = prediction; invalid voxels):
        the one device->host read"""
        C = self.n_classes
        if self.counts is None:
            return np.zeros((C, C), dtype=np.int64), 0
        c = self.counts.cpu().numpy()
        return c[:C * C].reshape(C, C), int(c[C * C])

    def get_stats(self):
        """the reference's dict: precision, recall and IoU of the completion (empty vs occupied) and the per-class
        IoU `iou_ssc` with its mean over classes 1.. `iou_ssc_mean`.  Raises ValueError when a counted voxel had a
        label outside [0, n_classes) other than 255, or a prediction outside [0, n_classes)."""
        hist, invalid = self.confusion()
        if invalid:
            raise ValueError("SSCMetrics: %d voxels had a label other than 255 outside [0, %d) or a prediction outside "
                             "it" % (invalid, self.n_classes))
        return stats_from_confusion(hist)


def counts_from_confusion(hist):
    """the reference's accumulators from a confusion matrix (rows = label, columns = prediction, 255 excluded):
    (tps, fps, fns) per class as int64 arrays and the completion tp, fp, fn as ints"""
    hist = np.asarray(hist, dtype=np.int64)
    tp = np.diag(hist).copy()
    fp = hist.sum(0) - tp
    fn = hist.sum(1) - tp
    c_tp = int(hist[1:, 1:].sum())      # occupied and predicted occupied
    c_fp = int(hist[0, 1:].sum())       # empty, predicted occupied
    c_fn = int(hist[1:, 0].sum())       # occupied, predicted empty
    return tp, fp, fn, c_tp, c_fp, c_fn


def stats_from_confusion(hist):
    """SSCMetrics.get_stats of the reference (loss/sscMetrics.py:93-109) from the same integer counts, with its
    types: Python floats (or int 0) for the completion, float64 numpy for the per-class IoU"""
    tp, fp, fn, c_tp, c_fp, c_fn = counts_from_confusion(hist)
    if c_tp != 0:
        precision = c_tp / (c_tp + c_fp)
        recall = c_tp / (c_tp + c_fn)
        iou = c_tp / (c_tp + c_fp + c_fn)
    else:
        precision, recall, iou = 0, 0, 0
    tps, fps, fns = (np.zeros(len(tp)) + v for v in (tp, fp, fn))       # the reference's float64 accumulators
    iou_ssc = tps / (tps + fps + fns + 1e-5)
    return {"precision": precision, "recall": recall, "iou": iou, "iou_ssc": iou_ssc,
            "iou_ssc_mean": np.mean(iou_ssc[1:])}
