"""Segmentation metrics whose counters live on the GPU: drop-ins for PyTorch-Encoding's `encoding.utils` metric functions
(ADE20K pixAcc / mIoU, test_lseg.py:314-395) and for the few-shot `Evaluator.classify_prediction` / `AverageMeter`
(mIoU / FB-IoU, test_lseg_zs.py:290-316; fewshot_data/common/evaluation.py, common/logger.py).

Every metric here reduces to one per-pixel rule over integer counters. Write p for the predicted class (the first maximal
class, as torch.max(output, 1)[1] picks it) and t for the int64 target; each pixel updates the counter row g of its image
(row 0 for SegmentationMetric, the class id for the few-shot meter), nclass being the number of metric classes:

    t < 0                : ignored (no counter changes)
    otherwise            : labeled[g] += 1
      p == t             : correct[g] += 1;  if t < nclass: inter[g][t] += 1
      0 <= p < nclass    : pred[g][p]  += 1
      t < nclass         : label[g][t] += 1
    union = pred + label - inter      (formed when read, never stored)

A row is int64 [inter(nclass) | pred(nclass) | label(nclass) | correct | labeled] (include/lseg_b200.h). The kernels add
to the rows; the only host synchronisation is where a result is read (get(), get_all(), the batch_* functions).

encoding.utils semantics (PyTorch-Encoding's encoding/utils/metrics.py, restated): predict = argmax + 1, target =
target + 1, predict *= (target > 0), then np.histogram(., bins=nclass, range=(1, nclass)) of the intersection, prediction
and target; pixel_labeled = sum(target > 0), pixel_correct = sum((predict == target) * (target > 0)). Hence a target
>= nclass (e.g. 255) counts as labeled and adds to `pred` but never to `label`, and a prediction >= nclass (K > nclass)
is dropped from the histograms. get() returns pixAcc = correct / (spacing(1) + labeled) and mIoU = mean over ALL nclass
classes of inter / (spacing(1) + union) (a class with zero union counts as 0).

Few-shot semantics (classify_prediction): K = nclass = 2. Without query_ignore_idx a gt == 255 pixel counts toward `pred`
only (t = 255 >= nclass); with it, the ignored positions and every gt == 255 pixel become t = -1 (the reference sets
pred_mask = 255 there, which histc(min=0, max=1) drops). compute_iou() keeps iou = inter / max(union, 1) over
class_ids_interest, mIoU = 100 * mean(iou[1]) and FB-IoU = 100 * mean_c(sum inter_c / sum union_c).

An image whose row id lies outside [0, rows) (a class_info beyond FewShotMeter's nclass, where the reference's index_add_
would fail) is not counted; the kernel records it on the device and FewShotMeter.compute_iou() raises on that record
(lseg_read_watchdog, tag 78). The record belongs to the device, not to one meter: it is raised by the next
compute_iou() on that device.

The validation loss (SegmentationLosses here, LSegNet.loss / LSegNetZS.loss fused into the output kernel) is
CrossEntropyLoss(ignore_index) with mean reduction: per pixel (m + log s) - v_t in fp32 over the classes' logits
(include/lseg_b200.h, section "cross-entropy"), summed in fp64 in a fixed order, so a call gives the same bits every time.
A target outside [0, K) other than ignore_index, where torch's CUDA kernel asserts and ends the process's CUDA context,
makes the loss NaN and is recorded on the device (tag 79); FewShotMeter.compute_iou() raises on that record.

Differences from the reference classes: the counters are int64 (the reference's float32 AverageMeter buffers round above
2^24 pixels per class) and are converted only when read; classify_prediction does not modify its arguments (the reference
writes 255 into pred_mask and multiplies query_ignore_idx in place) and returns int64 counts; everything runs on CUDA only.
"""
import numpy as np
import torch

from . import ops


SEGSTATS_TAG = 78  # lseg_read_watchdog tag of an image skipped for a row id outside [0, rows)
XENT_TAG = 79  # lseg_read_watchdog tag of a loss target outside [0, K) that is not ignore_index


def _raise_on_device_error(device):
    """Reads (and clears) the device's error record; raises when an image was skipped or a barrier timed out."""
    with torch.cuda.device(device):
        wd = ops.read_watchdog()
    if wd[0] == SEGSTATS_TAG:
        raise RuntimeError(f"a metric update skipped image {wd[1]} of its batch: its row id {wd[2]} is outside [0, {wd[3]}) "
                           f"(class_info beyond the meter's nclass?); the counters miss that image")
    if wd[0] == XENT_TAG:
        raise RuntimeError(f"a loss call met target {wd[3]} at pixel {wd[2]} (y * W + x) of image {wd[1]} of its batch: "
                           f"outside [0, K) and not ignore_index; that loss is NaN")
    if wd[0] != 0:
        raise RuntimeError(f"a kernel's barrier watchdog fired on {device} (tag {wd[0]}): results since the last check are "
                           f"not trustworthy")


def _row_len(nclass):
    return 3 * nclass + 2


def _split(row, nclass):
    """one counter row (numpy int64) -> (inter, union, correct, labeled)"""
    inter = row[:nclass]
    union = row[nclass:2 * nclass] + row[2 * nclass:3 * nclass] - inter
    return inter, union, row[3 * nclass], row[3 * nclass + 1]


def _as_target(target, device, shape):
    """int64 [B,H,W] target on `device`; an [H,W] target stands for a batch of one (test_lseg.py passes per-image
    targets without a batch dimension). A CPU target is copied."""
    t = torch.as_tensor(target)
    if t.dim() == len(shape) - 1:
        t = t.unsqueeze(0)
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"target has shape {tuple(torch.as_tensor(target).shape)}, expected {tuple(shape)}")
    return t.to(device=device, dtype=torch.int64).contiguous()


def _accumulate(stats, nclass, output, target, group=None):
    """Adds the counters of one prediction (scores [B,K,H,W] fp32/fp16, or an int64 mask [B,H,W]) to stats."""
    if not output.is_cuda:
        raise ValueError("lseg_b200.metrics runs on CUDA only: the prediction must be a CUDA tensor")
    if output.dim() == 4 and output.is_floating_point():
        if output.dtype != torch.float32:
            output = output.float()  # fp16 -> fp32 is exact: same first maximum
        output = output.contiguous()
        t = _as_target(target, output.device, (output.shape[0],) + tuple(output.shape[2:]))
        ops.seg_stats_scores(output, t, stats, nclass, group=group)
    elif output.dim() == 3 and not output.is_floating_point():
        output = output.to(torch.int64).contiguous()
        t = _as_target(target, output.device, tuple(output.shape))
        ops.seg_stats_mask(output, t, stats, nclass, group=group)
    else:
        raise ValueError(f"prediction must be scores [B,K,H,W] (float) or a class mask [B,H,W] (integer), got "
                         f"{output.dtype} {tuple(output.shape)}")
    return stats


def _mean_loss(acc):
    """0-d fp32 mean of a loss accumulator {sum, count} (float64 [2]); NaN when every pixel was ignored, as in torch."""
    return (acc[0] / acc[1]).float()


class SegmentationLosses:
    """PyTorch-Encoding's SegmentationLosses (the criterion of LSegmentationModule.get_criterion) for what LSeg uses
    of it: with se_loss = aux = False and no class weight it is CrossEntropyLoss(ignore_index) with mean reduction,
    computed here by one device kernel over the fp32 scores [B,K,H,W] without torch's log_softmax intermediate. The loss
    terms LSeg never produces inputs for (se_loss, aux, class weights) raise NotImplementedError. A target outside
    [0, K) other than ignore_index gives NaN and a device record (lseg_read_watchdog tag 79) where torch would assert."""

    def __init__(self, se_loss=False, se_weight=0.2, nclass=-1, aux=False, aux_weight=0.4, weight=None,
                 ignore_index=-1):
        if se_loss:
            raise NotImplementedError("se_loss: LSeg's net returns no SE-loss prediction")
        if aux:
            raise NotImplementedError("aux: LSeg's net returns no auxiliary output")
        if weight is not None:
            raise NotImplementedError("class weights are not supported")
        self.se_loss, self.aux = se_loss, aux
        self.nclass = nclass
        self.se_weight, self.aux_weight = se_weight, aux_weight
        self.ignore_index = int(ignore_index)

    def __call__(self, *inputs):
        if len(inputs) != 2:
            raise ValueError(f"SegmentationLosses takes (scores, target), got {len(inputs)} arguments")
        scores, target = inputs
        if not scores.is_cuda:
            raise ValueError("lseg_b200.metrics runs on CUDA only: the scores must be a CUDA tensor")
        if scores.dim() != 4 or not scores.is_floating_point():
            raise ValueError(f"scores must be float [B,K,H,W], got {scores.dtype} {tuple(scores.shape)}")
        scores = scores.float().contiguous()
        t = _as_target(target, scores.device, (scores.shape[0],) + tuple(scores.shape[2:]))
        acc = torch.zeros(2, dtype=torch.float64, device=scores.device)
        ops.xent_scores(scores, t, acc, self.ignore_index)
        return _mean_loss(acc)

    forward = __call__


def _batch_row(output, target, nclass):
    stats = torch.zeros((1, _row_len(nclass)), dtype=torch.int64, device=output.device)
    _accumulate(stats, nclass, output, target)
    return stats[0].cpu().numpy()


def batch_pix_accuracy(output, target):
    """encoding.utils.batch_pix_accuracy: (pixel_correct, pixel_labeled) of torch.max(output, 1)[1] against target."""
    row = _batch_row(output, target, 1)  # correct / labeled do not depend on nclass
    return row[3], row[4]


def batch_intersection_union(output, target, nclass):
    """encoding.utils.batch_intersection_union: (area_inter, area_union), int64 numpy arrays [nclass]."""
    inter, union, _, _ = _split(_batch_row(output, target, nclass), nclass)
    return inter, union


class SegmentationMetric:
    """encoding.utils.SegmentationMetric with its counters on the GPU: update() enqueues one kernel and never
    synchronises; get() / get_all() copy the nclass x 3 + 2 counters to the host."""

    def __init__(self, nclass, device=None):
        self.nclass = int(nclass)
        if self.nclass <= 0:
            raise ValueError(f"nclass={nclass} must be positive")
        self.device = torch.device(device) if device is not None else None
        self.stats = None  # int64 [1, 3*nclass+2], allocated on the device of the first update unless `device` is given
        if self.device is not None:
            self._buffer(self.device)

    def _buffer(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("lseg_b200.metrics runs on CUDA only")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if self.stats is None:
            self.stats = torch.zeros((1, _row_len(self.nclass)), dtype=torch.int64, device=device)
        elif self.stats.device != device:
            raise ValueError(f"prediction is on {device}, the metric's counters are on {self.stats.device}")
        return self.stats

    def update(self, labels, preds):
        """preds: scores [B,K,H,W] (fp32 / fp16) or an int64 class mask [B,H,W], or a list / tuple of them paired with
        `labels`; labels: int64 [B,H,W] (or [H,W] for a batch of one), on any device."""
        if isinstance(preds, torch.Tensor):
            _accumulate(self._buffer(preds.device), self.nclass, preds, labels)
        elif isinstance(preds, (list, tuple)):
            for label, pred in zip(labels, preds):
                _accumulate(self._buffer(pred.device), self.nclass, pred, label)
        else:
            raise NotImplementedError

    def _row(self):
        if self.stats is None:
            return np.zeros(_row_len(self.nclass), dtype=np.int64)
        return self.stats[0].cpu().numpy()

    def get(self):
        inter, union, correct, labeled = _split(self._row(), self.nclass)
        pixAcc = 1.0 * correct / (np.spacing(1) + labeled)
        IoU = 1.0 * inter / (np.spacing(1) + union)
        mIoU = IoU.mean()
        return pixAcc, mIoU

    def get_all(self):
        inter, union, correct, labeled = _split(self._row(), self.nclass)
        return correct, labeled, inter, union

    def reset(self):
        if self.stats is not None:
            self.stats.zero_()


def _fewshot_target(gt_mask, query_ignore_idx):
    t = gt_mask.to(torch.int64)
    if query_ignore_idx is not None:
        drop = (query_ignore_idx.to(t.device) != 0) | (t == 255)
        t = torch.where(drop, torch.full_like(t, -1), t)
    return t.contiguous()


def classify_prediction(pred_mask, gt_mask, query_ignore_idx=None):
    """Evaluator.classify_prediction: (area_inter, area_union), each int64 [2, B], of binary masks [B,H,W]. Unlike the
    reference it leaves pred_mask and query_ignore_idx unchanged."""
    if not pred_mask.is_cuda:
        raise ValueError("lseg_b200.metrics runs on CUDA only: pred_mask must be a CUDA tensor")
    B = pred_mask.shape[0]
    stats = torch.zeros((B, _row_len(2)), dtype=torch.int64, device=pred_mask.device)
    t = _fewshot_target(gt_mask.to(pred_mask.device), query_ignore_idx)
    _accumulate(stats, 2, pred_mask, t, group=torch.arange(B, device=pred_mask.device))
    inter = stats[:, 0:2]
    union = stats[:, 2:4] + stats[:, 4:6] - inter
    return inter.t(), union.t()


class FewShotMeter:
    """AverageMeter's counting part (update / compute_iou; not its Logger-based write_process / write_result) with int64
    counters: one counter row per class id, nclass rows of the K = 2 layout, which LSegNetZS.update_metric accumulates
    into directly (row = class_info[b]). update() adds inter into the `inter` and `label` columns and union into the `pred` columns, so
    pred + label - inter reads back as the union however the two kinds of updates are mixed."""

    def __init__(self, nclass, class_ids, device=None):
        self.nclass = int(nclass)
        device = torch.device(device if device is not None else "cuda")
        if device.type != "cuda":
            raise ValueError("lseg_b200.metrics runs on CUDA only")
        self.class_ids_interest = torch.as_tensor(class_ids, dtype=torch.int64).to(device)
        self.stats = torch.zeros((self.nclass, _row_len(2)), dtype=torch.int64, device=device)
        self.loss_buf = []  # one loss per update (LSegNetZS.loss with meter= appends its own)

    @property
    def intersection_buf(self):
        return self.stats[:, 0:2].t()

    @property
    def union_buf(self):
        return (self.stats[:, 2:4] + self.stats[:, 4:6] - self.stats[:, 0:2]).t()

    def update(self, inter_b, union_b, class_id, loss=None):
        """Adds [2, B] counts to the rows class_id [B] (AverageMeter.update's index_add_) and appends `loss` to loss_buf
        (torch.tensor(0.0) for None, as AverageMeter does)."""
        self.loss_buf.append(torch.tensor(0.0) if loss is None else loss)
        cid = torch.as_tensor(class_id).to(device=self.stats.device, dtype=torch.int64).reshape(-1)
        inter = inter_b.to(device=self.stats.device, dtype=torch.int64).t()
        union = union_b.to(device=self.stats.device, dtype=torch.int64).t()
        self.stats[:, 0:2].index_add_(0, cid, inter)
        self.stats[:, 2:4].index_add_(0, cid, union)
        self.stats[:, 4:6].index_add_(0, cid, inter)

    def compute_iou(self):
        """(mIoU, FB-IoU) in percent, float64 0-d tensors, formed from the exact counts. Synchronises, and raises if an
        update since the last check skipped an image for a class id outside [0, nclass)."""
        _raise_on_device_error(self.stats.device)
        inter = self.intersection_buf.double()
        union = self.union_buf.double()
        iou = inter / torch.clamp(union, min=1.0)
        iou = iou.index_select(1, self.class_ids_interest)
        miou = iou[1].mean() * 100
        fb_iou = (inter.index_select(1, self.class_ids_interest).sum(dim=1) /
                  union.index_select(1, self.class_ids_interest).sum(dim=1)).mean() * 100
        return miou, fb_iou

    def reset(self):
        self.stats.zero_()
        self.loss_buf = []
