"""CPU references for the segmentation metric counters (lseg_b200.metrics, include/lseg_b200.h).

rule_counts is the per-pixel rule as written in the spec; encoding_* restate PyTorch-Encoding's
encoding/utils/metrics.py (predict = argmax + 1, target = target + 1, predict *= (target > 0), np.histogram with
bins=nclass, range=(1, nclass)); fewshot_target maps classify_prediction's ignore handling onto the rule's t < 0.
tests/test_metrics_cpu.py checks them against each other and against the unmodified reference few-shot code's outputs;
tests/test_metrics_gpu.py holds the kernels to rule_counts exactly.
"""
import numpy as np


def row_len(nclass):
    return 3 * nclass + 2


def rule_counts(pred, target, nclass, group=None, G=1):
    """pred, target: integer arrays [B, ...]; group: ids [B] (None: all row 0). -> int64 [G, 3*nclass+2]:
    [inter | pred | label | correct | labeled] per row. Images whose group is outside [0, G) are skipped."""
    pred = np.asarray(pred, dtype=np.int64)
    target = np.asarray(target, dtype=np.int64)
    out = np.zeros((G, row_len(nclass)), dtype=np.int64)
    for b in range(pred.shape[0]):
        g = 0 if group is None else int(group[b])
        if not 0 <= g < G:
            continue
        p = pred[b].reshape(-1)
        t = target[b].reshape(-1)
        keep = t >= 0
        p, t = p[keep], t[keep]
        hit = p == t
        out[g, :nclass] += np.bincount(t[hit & (t < nclass)], minlength=nclass)
        out[g, nclass:2 * nclass] += np.bincount(p[(p >= 0) & (p < nclass)], minlength=nclass)
        out[g, 2 * nclass:3 * nclass] += np.bincount(t[t < nclass], minlength=nclass)
        out[g, 3 * nclass] += int(hit.sum())
        out[g, 3 * nclass + 1] += int(t.size)
    return out


def split(row, nclass):
    """one counter row -> (inter, union, correct, labeled)"""
    inter = row[:nclass]
    return inter, row[nclass:2 * nclass] + row[2 * nclass:3 * nclass] - inter, row[3 * nclass], row[3 * nclass + 1]


def first_argmax(scores):
    """torch.max(scores, 1)[1] of NaN-free scores [B, K, ...] (numpy's argmax also returns the first maximum)."""
    return np.argmax(np.asarray(scores), axis=1)


def encoding_batch_pix_accuracy(predict_idx, target):
    """encoding.utils.batch_pix_accuracy after its torch.max: predict_idx = argmax [B, H, W]."""
    predict = np.asarray(predict_idx).astype("int64") + 1
    target = np.asarray(target).astype("int64") + 1
    pixel_labeled = np.sum(target > 0)
    pixel_correct = np.sum((predict == target) * (target > 0))
    return pixel_correct, pixel_labeled


def encoding_batch_intersection_union(predict_idx, target, nclass):
    """encoding.utils.batch_intersection_union after its torch.max."""
    mini, maxi, nbins = 1, nclass, nclass
    predict = np.asarray(predict_idx).astype("int64") + 1
    target = np.asarray(target).astype("int64") + 1
    predict = predict * (target > 0).astype(predict.dtype)
    intersection = predict * (predict == target)
    area_inter, _ = np.histogram(intersection, bins=nbins, range=(mini, maxi))
    area_pred, _ = np.histogram(predict, bins=nbins, range=(mini, maxi))
    area_lab, _ = np.histogram(target, bins=nbins, range=(mini, maxi))
    area_union = area_pred + area_lab - area_inter
    return area_inter, area_union


class EncodingMetric:
    """encoding.utils.SegmentationMetric over argmax masks (update / get / get_all)."""

    def __init__(self, nclass):
        self.nclass = nclass
        self.total_inter = 0
        self.total_union = 0
        self.total_correct = 0
        self.total_label = 0

    def update(self, target, predict_idx):
        correct, labeled = encoding_batch_pix_accuracy(predict_idx, target)
        inter, union = encoding_batch_intersection_union(predict_idx, target, self.nclass)
        self.total_correct += correct
        self.total_label += labeled
        self.total_inter += inter
        self.total_union += union

    def get(self):
        pixAcc = 1.0 * self.total_correct / (np.spacing(1) + self.total_label)
        IoU = 1.0 * self.total_inter / (np.spacing(1) + self.total_union)
        return pixAcc, IoU.mean()

    def get_all(self):
        return self.total_correct, self.total_label, self.total_inter, self.total_union


def fewshot_target(gt, ignore=None):
    """classify_prediction's targets under the rule: with query_ignore_idx, ignored positions and gt == 255 become -1."""
    t = np.asarray(gt).astype(np.int64)
    if ignore is not None:
        t = np.where((np.asarray(ignore) != 0) | (t == 255), -1, t)
    return t


def fewshot_iou(inter_buf, union_buf, class_ids):
    """AverageMeter.compute_iou on [2, n_classes] buffers -> (mIoU, FB-IoU) in percent, float64."""
    inter = np.asarray(inter_buf, dtype=np.float64)[:, class_ids]
    union = np.asarray(union_buf, dtype=np.float64)[:, class_ids]
    iou = inter / np.maximum(union, 1.0)
    return iou[1].mean() * 100, (inter.sum(1) / union.sum(1)).mean() * 100
