"""CPU checks of the segmentation metric spec (lseg_b200.metrics): the per-pixel counter rule equals a restatement of
PyTorch-Encoding's metric functions (np.histogram exactly as encoding calls it) on awkward inputs, and reproduces the
unmodified reference few-shot Evaluator / AverageMeter outputs committed in tests/golden/ref_metrics_fss.npz."""
import os

import numpy as np
import pytest

from segstats_oracle import (EncodingMetric, encoding_batch_intersection_union, encoding_batch_pix_accuracy,
                             fewshot_iou, fewshot_target, row_len, rule_counts, split)

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _awkward(rng, B, H, W, K, nclass):
    """predictions in [0, K) with K > nclass, targets mixing -5, -1, every class, nclass, nclass + 7 and 255"""
    pred = rng.integers(0, K, size=(B, H, W))
    specials = np.array([-5, -1, nclass, nclass + 7, 255])
    t = rng.integers(0, nclass, size=(B, H, W))
    pick = rng.random((B, H, W))
    t = np.where(pick < 0.25, specials[rng.integers(0, len(specials), size=(B, H, W))], t)
    t = np.where(pick > 0.6, pred, t)  # plenty of hits, including hits on classes >= nclass
    return pred, t


@pytest.mark.parametrize("nclass", [1, 2, 150, 512])
def test_rule_matches_encoding(nclass):
    rng = np.random.default_rng(nclass)
    K = nclass + 3
    metric = EncodingMetric(nclass)
    total = np.zeros(row_len(nclass), dtype=np.int64)
    for step in range(3):
        pred, t = _awkward(rng, 2, 23 + step, 31, K, nclass)
        row = rule_counts(pred, t, nclass)[0]
        inter, union, correct, labeled = split(row, nclass)
        e_inter, e_union = encoding_batch_intersection_union(pred, t, nclass)
        e_correct, e_labeled = encoding_batch_pix_accuracy(pred, t)
        np.testing.assert_array_equal(inter, e_inter)
        np.testing.assert_array_equal(union, e_union)
        assert (correct, labeled) == (e_correct, e_labeled)
        metric.update(t, pred)
        total += row
    inter, union, correct, labeled = split(total, nclass)
    g_correct, g_labeled, g_inter, g_union = metric.get_all()
    assert (correct, labeled) == (g_correct, g_labeled)
    np.testing.assert_array_equal(inter, g_inter)
    np.testing.assert_array_equal(union, g_union)
    pix_acc, miou = metric.get()
    assert pix_acc == 1.0 * correct / (np.spacing(1) + labeled)
    assert miou == (1.0 * inter / (np.spacing(1) + union)).mean()


def test_rule_quirks():
    """The encoding quirks the spec keeps, on hand-made pixels (nclass = 3)."""
    pred = np.array([[[0, 1, 2, 4, 1, 2]]])
    t = np.array([[[0, -1, 255, 4, 3, -5]]])
    inter, union, correct, labeled = split(rule_counts(pred, t, 3)[0], 3)
    assert labeled == 4 and correct == 2          # t = 255 and t = 3 are labeled; p == t == 4 is correct
    np.testing.assert_array_equal(inter, [1, 0, 0])
    np.testing.assert_array_equal(union, [1, 1, 1])  # 255 / 3 add to pred only, p = 4 >= nclass to nothing
    np.testing.assert_array_equal(encoding_batch_intersection_union(pred, t, 3), (inter, union))


def test_rule_groups():
    rng = np.random.default_rng(7)
    pred, t = _awkward(rng, 5, 9, 11, 6, 4)
    group = np.array([2, 0, 2, 9, -1])  # repeated, sparse, and two out of range (skipped)
    got = rule_counts(pred, t, 4, group=group, G=3)
    want = np.zeros_like(got)
    for b, g in enumerate(group):
        if 0 <= g < 3:
            want[g] += rule_counts(pred[b:b + 1], t[b:b + 1], 4)[0]
    np.testing.assert_array_equal(got, want)
    assert not got[1].any()


def test_fewshot_rule_matches_reference_golden():
    """The rule with classify_prediction's target mapping reproduces the unmodified reference Evaluator and AverageMeter
    (oracle/make_golden_metrics.py): per-batch [2, B] areas, the meter's buffers and its mIoU / FB-IoU."""
    gold = np.load(os.path.join(GOLD, "ref_metrics_fss.npz"))
    n_classes = int(gold["n_classes"])
    rows = np.zeros((n_classes, row_len(2)), dtype=np.int64)
    saw_empty = saw_255 = False
    for i in range(gold["pred"].shape[0]):
        pred = gold["pred"][i].astype(np.int64)
        gt = gold["gt"][i].astype(np.int64)
        ignore = gold["ignore"][i] if gold["has_ignore"][i] else None
        t = fewshot_target(gt, ignore)
        B = pred.shape[0]
        per_image = rule_counts(pred, t, 2, group=np.arange(B), G=B)
        inter = per_image[:, 0:2].T
        union = (per_image[:, 2:4] + per_image[:, 4:6] - per_image[:, 0:2]).T
        np.testing.assert_array_equal(inter, gold["area_inter"][i])
        np.testing.assert_array_equal(union, gold["area_union"][i])
        rows += rule_counts(pred, t, 2, group=gold["class_id"][i], G=n_classes)
        saw_empty |= bool((inter.sum(0) == 0).any())
        saw_255 |= bool((gt == 255).any())
    assert saw_empty and saw_255 and gold["has_ignore"].any() and not gold["has_ignore"].all()
    inter_buf = rows[:, 0:2].T
    union_buf = (rows[:, 2:4] + rows[:, 4:6] - rows[:, 0:2]).T
    np.testing.assert_array_equal(inter_buf, gold["intersection_buf"])
    np.testing.assert_array_equal(union_buf, gold["union_buf"])
    miou, fb_iou = fewshot_iou(inter_buf, union_buf, gold["class_ids"])
    # the reference forms these in float32 from float32 buffers; the counts here are exact
    assert miou == pytest.approx(float(gold["miou"]), rel=1e-6)
    assert fb_iou == pytest.approx(float(gold["fb_iou"]), rel=1e-6)
