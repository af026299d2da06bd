"""TEST INFRASTRUCTURE. Golden vectors for the few-shot metrics (lseg_b200.metrics.classify_prediction / FewShotMeter).

Runs the UNMODIFIED reference `fewshot_data/common/evaluation.py::Evaluator.classify_prediction` and
`fewshot_data/common/logger.py::AverageMeter.update / compute_iou` on seeded synthetic binary masks, on CPU, and stores
the masks, class ids and every result in tests/golden/ref_metrics_fss.npz. Three shims make the reference run on CPU
here, in the way oracle/ref_standins.py stands in for absent packages; none changes what the reference computes:
  * `tensorboardX` (imported by logger.py, used only by its Logger class) is an empty stand-in module;
  * `torch.Tensor.cuda` is the identity (AverageMeter hard-codes .cuda() on its buffers);
  * `torch.histc` casts its input to float32 first (CPU histc has no int64 kernel; the masks hold 0, 1 and 255, which
    float32 represents exactly).
Cases: batches with and without query_ignore_idx, gt == 255 pixels in both, and an all-wrong image with no 255 / ignored
pixel, so classify_prediction takes its empty-intersection branch.

    LSEG_REFERENCE_ROOT=<lang-seg checkout> python oracle/make_golden_metrics.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LSEG_REFERENCE_ROOT", "")

N_BATCH, B, H, W = 6, 4, 37, 29
N_CLASSES = 20                  # AverageMeter's row count for benchmark 'pascal'
CLASS_IDS = [5, 6, 7, 8, 9]     # a PASCAL-5i fold's class ids: compute_iou reads these rows only


def masks(g, with_ignore):
    gt = (torch.rand(B, H, W, generator=g) < 0.4).long()
    pred = torch.where(torch.rand(B, H, W, generator=g) < 0.7, gt, 1 - gt)
    gt[torch.rand(B, H, W, generator=g) < 0.05] = 255
    ignore = torch.zeros(B, H, W, dtype=torch.long)
    if with_ignore:  # the reference asserts ignore & gt == 0, so only background pixels can be ignored
        ignore = ((torch.rand(B, H, W, generator=g) < 0.1) & (gt == 0)).long()
    # image 0: every prediction wrong and no 255 / ignored pixel -> empty intersection branch
    gt[0] = (torch.rand(H, W, generator=g) < 0.5).long()
    pred[0] = 1 - gt[0]
    ignore[0] = 0
    return pred, gt, ignore


def main():
    if not REF or not os.path.isdir(os.path.join(REF, "fewshot_data")):
        raise SystemExit("set LSEG_REFERENCE_ROOT to a lang-seg checkout")
    sys.path.insert(0, REF)
    tbx = types.ModuleType("tensorboardX")
    tbx.SummaryWriter = object
    sys.modules.setdefault("tensorboardX", tbx)
    torch.Tensor.cuda = lambda self, *a, **k: self
    histc = torch.histc
    torch.histc = lambda x, *a, **k: histc(x.float(), *a, **k)
    from fewshot_data.common.evaluation import Evaluator
    from fewshot_data.common.logger import AverageMeter

    Evaluator.initialize()
    meter = AverageMeter(types.SimpleNamespace(benchmark="pascal", class_ids=CLASS_IDS))
    g = torch.Generator().manual_seed(2024)
    out = {k: [] for k in ("pred", "gt", "ignore", "has_ignore", "class_id", "area_inter", "area_union")}
    for i in range(N_BATCH):
        with_ignore = i % 2 == 1
        pred, gt, ignore = masks(g, with_ignore)
        class_id = torch.tensor(CLASS_IDS)[torch.randint(0, len(CLASS_IDS), (B,), generator=g)]
        # the reference writes into pred_mask and query_ignore_idx: hand it copies
        inter, union = Evaluator.classify_prediction(pred.clone(), gt.clone(), ignore.clone() if with_ignore else None)
        meter.update(inter, union, class_id, loss=None)
        for k, v in (("pred", pred), ("gt", gt), ("ignore", ignore), ("class_id", class_id)):
            out[k].append(v.numpy().astype(np.uint8 if k != "class_id" else np.int64))
        out["has_ignore"].append(with_ignore)
        out["area_inter"].append(inter.double().numpy().astype(np.int64))
        out["area_union"].append(union.double().numpy().astype(np.int64))
    miou, fb_iou = meter.compute_iou()
    res = {k: np.stack(v) for k, v in out.items()}
    res.update(intersection_buf=meter.intersection_buf.numpy().astype(np.int64),
               union_buf=meter.union_buf.numpy().astype(np.int64), miou=np.float64(miou.item()),
               fb_iou=np.float64(fb_iou.item()), n_classes=np.int64(N_CLASSES), class_ids=np.array(CLASS_IDS))
    path = os.path.join(ROOT, "tests", "golden", "ref_metrics_fss.npz")
    np.savez_compressed(path, **res)
    print(f"wrote {path}: miou {res['miou']:.4f} fb_iou {res['fb_iou']:.4f}, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
