"""GPU checks of the segmentation metric counters (csrc/segstats.cuh, the fused output stage of csrc/elementwise.cuh,
lseg_b200.metrics). Every comparison is exact integer equality against the per-pixel rule of tests/segstats_oracle.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity_util import NET_KW, state_dict, synth
from segstats_oracle import EncodingMetric, first_argmax, fewshot_target, fewshot_iou, row_len, rule_counts, split

pytestmark = pytest.mark.gpu
SMEM_MAX_CLASS = 1364  # kSegSmemMaxClass: above it the kernels count with global atomics


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops
    ops.read_watchdog()  # start from a clear error record
    return ops


def _no_error(ops):
    wd = ops.read_watchdog()
    assert wd[0] == 0, f"watchdog / metric error record set: {wd}"


def _targets(g, shape, nclass, pred=None):
    """int64 targets: every class, plus -1, -5, 255 and nclass; copies of `pred` on ~40 % of the pixels"""
    t = torch.randint(0, nclass, shape, generator=g)
    r = torch.rand(shape, generator=g)
    specials = torch.tensor([-1, -5, 255, nclass])
    t = torch.where(r < 0.15, specials[torch.randint(0, 4, shape, generator=g)], t)
    if pred is not None:
        t = torch.where(r > 0.6, pred.cpu(), t)
    return t


def _prefilled(G, nclass, base):
    """counters pre-filled near a 32-bit boundary: the kernels must add to them without wrapping"""
    return torch.full((G, row_len(nclass)), base, dtype=torch.int64) + torch.arange(G * row_len(nclass)).view(G, -1)


SCORE_CASES = [  # (B, K, H, W, nclass, groups, G)
    (1, 5, 7, 9, 5, None, 1),
    (8, 150, 13, 17, 150, None, 1),                 # odd H*W, B = 8
    (3, 40, 31, 33, 20, [2, 0, 2], 4),               # K > nclass, repeated and sparse groups
    (4, 7, 45, 45, 3, [1, 1, 1, 1], 2),              # several blocks per image
    (2, 3, 16, 18, SMEM_MAX_CLASS, [0, 1], 2),       # largest shared-memory histogram
    (2, 3, 16, 18, SMEM_MAX_CLASS + 1, [1, 0], 2),   # global-atomic counting
]


@pytest.mark.parametrize("base", [0, 2 ** 31 - 5, 2 ** 32 - 3])
@pytest.mark.parametrize("case", SCORE_CASES, ids=[f"B{c[0]}K{c[1]}_{c[2]}x{c[3]}_n{c[4]}" for c in SCORE_CASES])
def test_seg_stats_kernels(ops, case, base):
    B, K, H, W, nclass, groups, G = case
    g = torch.Generator().manual_seed(B * 1000 + K + H)
    scores = torch.randn(B, K, H, W, generator=g)
    # ties: a quarter of the pixels get their maximum planted at two classes (the first must win), some +-inf
    r = torch.rand(B, H, W, generator=g)
    ka = torch.randint(0, K, (B, H, W), generator=g)
    kb = torch.randint(0, K, (B, H, W), generator=g)
    top = scores.max(1, keepdim=True).values + 1.0
    tie = (r < 0.25).unsqueeze(1)
    for kk in (ka.unsqueeze(1), kb.unsqueeze(1)):
        scores.scatter_(1, kk, torch.where(tie, top, scores.gather(1, kk)))
    scores[:, 0][r > 0.97] = -float("inf")
    scores[:, K - 1][(r > 0.95) & (r <= 0.96)] = float("inf")
    pred = torch.from_numpy(first_argmax(scores.numpy()))
    assert torch.equal(pred, torch.max(scores, 1)[1])
    target = _targets(g, (B, H, W), nclass, pred)
    group = torch.tensor(groups, dtype=torch.int32) if groups is not None else None
    want = rule_counts(pred.numpy(), target.numpy(), nclass, groups, G) + _prefilled(G, nclass, base).numpy()
    dev = "cuda"
    for run in ("scores", "mask"):
        stats = _prefilled(G, nclass, base).to(dev)
        gd = group.to(dev) if group is not None else None
        if run == "scores":
            ops.seg_stats_scores(scores.to(dev), target.to(dev), stats, nclass, group=gd)
        else:
            ops.seg_stats_mask(pred.to(dev), target.to(dev), stats, nclass, group=gd)
        got = stats.cpu().numpy()
        assert np.array_equal(got, want), (run, np.argwhere(got != want)[:5], got[got != want][:5], want[got != want][:5])
    _no_error(ops)


def test_seg_stats_accumulates(ops):
    g = torch.Generator().manual_seed(5)
    scores = torch.randn(2, 6, 20, 24, generator=g)
    target = _targets(g, (2, 20, 24), 6)
    stats = torch.zeros((1, row_len(6)), dtype=torch.int64, device="cuda")
    for _ in range(3):
        ops.seg_stats_scores(scores.cuda(), target.cuda(), stats, 6)
    want = 3 * rule_counts(first_argmax(scores.numpy()), target.numpy(), 6)
    assert np.array_equal(stats.cpu().numpy(), want)


def test_seg_stats_rejects_bad_arguments(ops):
    from lseg_b200 import _lib
    import ctypes as C
    lib = _lib.load()
    s = torch.zeros(2, row_len(4) + 1, dtype=torch.int64, device="cuda")
    sc = torch.zeros(1, 4, 8, 8, device="cuda")
    t = torch.zeros(1, 8, 8, dtype=torch.int64, device="cuda")
    p = C.c_void_p
    st = p(torch.cuda.current_stream().cuda_stream)
    cases = [
        ((None, p(t.data_ptr()), None, 1, 4, 8, 8, 4, 1, p(s.data_ptr()), st), "prediction"),
        ((p(sc.data_ptr()), None, None, 1, 4, 8, 8, 4, 1, p(s.data_ptr()), st), "target"),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 4, 8, 8, 4, 1, None, st), "stats"),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 4, 8, 8, 4, 1, p(s.data_ptr() + 4), st), "stats must be 8-byte"),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 4, 8, 8, 0, 1, p(s.data_ptr()), st), "nclass"),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 4, 8, 8, 4, 0, p(s.data_ptr()), st), "G="),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 0, 4, 8, 8, 4, 1, p(s.data_ptr()), st), "B="),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 70000, 4, 8, 8, 4, 1, p(s.data_ptr()), st), "B="),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 4, 0, 8, 4, 1, p(s.data_ptr()), st), "H="),
        ((p(sc.data_ptr()), p(t.data_ptr()), None, 1, 0, 8, 8, 4, 1, p(s.data_ptr()), st), "K="),
    ]
    before = s.clone()
    for args, word in cases:
        assert lib.lseg_seg_stats_scores(*args) != 0, word
        assert word in lib.lseg_last_error().decode(), (word, lib.lseg_last_error())
    assert lib.lseg_seg_stats_mask(p(t.data_ptr()), p(t.data_ptr()), None, 1, 8, 8, 4, 1, p(s.data_ptr() + 4), st) != 0
    assert "stats must be 8-byte" in lib.lseg_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(s, before)
    with pytest.raises(ValueError, match="stats must be int64"):
        ops.seg_stats_mask(t, t, s, 4)


def test_out_of_range_group_is_reported(ops):
    g = torch.Generator().manual_seed(9)
    pred = torch.randint(0, 3, (4, 10, 12), generator=g)
    target = _targets(g, (4, 10, 12), 3, pred)
    group = torch.tensor([0, 5, 1, -2], dtype=torch.int32)
    stats = torch.zeros((2, row_len(3)), dtype=torch.int64, device="cuda")
    ops.seg_stats_mask(pred.cuda(), target.cuda(), stats, 3, group=group.cuda())
    wd = ops.read_watchdog()
    assert wd[0] == 78 and wd[1] in (1, 3) and wd[2] in (5, -2) and wd[3] == 2, wd
    assert ops.read_watchdog()[0] == 0  # cleared by the read
    assert np.array_equal(stats.cpu().numpy(), rule_counts(pred.numpy(), target.numpy(), 3, group.numpy(), 2))


def test_group_length_must_match_batch(ops):
    pred = torch.zeros(4, 8, 8, dtype=torch.int64, device="cuda")
    stats = torch.zeros((2, row_len(3)), dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="group has 3 entries, the batch has 4"):
        ops.seg_stats_mask(pred, pred, stats, 3, group=torch.tensor([0, 1, 0], device="cuda"))
    assert not stats.any()


# ------------------------------------------------------------------------------------------------
# the fused output stage through the engine
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def net(ops):
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


def _check_update_metric(ops, net, x, tokens, nclass, seed):
    """update_metric == seg_stats_mask(predict(x)) == the rule; the engine's optional mask / logits outputs equal
    predict() / forward() bit for bit."""
    from lseg_b200.metrics import SegmentationMetric
    x = x.cuda()
    mask = net.predict(x, tokens)
    g = torch.Generator().manual_seed(seed)
    target = _targets(g, tuple(mask.shape), nclass, mask).cuda()
    metric = SegmentationMetric(nclass)
    net.update_metric(metric, x, target, tokens)
    ref = torch.zeros((1, row_len(nclass)), dtype=torch.int64, device="cuda")
    ops.seg_stats_mask(mask, target, ref, nclass)
    want = rule_counts(mask.cpu().numpy(), target.cpu().numpy(), nclass)
    assert np.array_equal(ref.cpu().numpy(), want)
    assert np.array_equal(metric.stats.cpu().numpy(), want)
    eng = net._engine_for(x.device)
    feats = net._text_features(eng, tokens)
    K = tokens.shape[0]
    stats = torch.zeros_like(ref)
    m2 = torch.full_like(mask, -7)
    logits = torch.empty((x.shape[0], K) + tuple(x.shape[2:]), device="cuda")
    eng.forward_stats(x, feats, K, target, stats, nclass, mask=m2, logits=logits)
    assert torch.equal(stats, ref) and torch.equal(m2, mask)
    assert torch.equal(logits, net(x, tokens))
    _no_error(ops)


@pytest.mark.parametrize("B,H,W,K,nclass", [
    (2, 480, 480, 150, 150),
    (2, 256, 384, 150, 150),                # H != W
    (1, 736, 736, 12, 12),                  # 2W > 512: the multi-pass column loop
    (2, 64, 96, 150, 100),                  # K > nclass
    (2, 64, 96, 20, SMEM_MAX_CLASS),        # largest shared-memory histogram
    (2, 64, 96, 20, SMEM_MAX_CLASS + 1),    # global-atomic counting
])
def test_update_metric_equals_mask_stats(ops, net, B, H, W, K, nclass):
    x = synth.make_image(B, H, W, seed=H + W + K)
    tokens = synth.tokenize(synth.ade20k_labels()[:K])
    _check_update_metric(ops, net, x, tokens, nclass, seed=B + H)


def test_update_metric_arch_option1(ops):
    from lseg_b200.lseg_net import LSegNet
    kw = dict(NET_KW, arch_option=1, block_depth=2, activation="lrelu")
    labels = synth.ade20k_labels()[:5]
    n = LSegNet(labels=labels, **kw)
    n.load_state_dict(synth.make_state_dict(0, head_block=True))
    n = n.cuda().eval()
    _check_update_metric(ops, n, synth.make_image(2, 64, 96, seed=11), synth.tokenize(labels), 5, seed=11)


@pytest.fixture(scope="module")
def zs(ops):
    from lseg_b200.lseg_net import LSegNetZS
    names = [f"class {i}" for i in range(20)]
    n = LSegNetZS(label_list=names, **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


@pytest.mark.parametrize("with_ignore", [False, True])
def test_zero_shot_update_metric(ops, zs, with_ignore):
    """K = 2, group = class_info; 473 x 473 images padded to 480 with a target padded with -1 give the counters of the
    cropped 473 x 473 mask."""
    from lseg_b200.metrics import FewShotMeter, classify_prediction
    B = 4
    x = F.pad(synth.make_image(B, 473, 473, seed=473), (0, 7, 0, 7), value=-1.0).cuda()
    class_info = torch.tensor([3, 7, 3, 19])
    mask = zs.predict(x, class_info.cuda())[:, :473, :473]
    g = torch.Generator().manual_seed(17)
    gt = torch.where(torch.rand(B, 473, 473, generator=g) < 0.3, 1 - mask.cpu(), mask.cpu())
    gt[torch.rand(B, 473, 473, generator=g) < 0.05] = 255
    ignore = ((torch.rand(B, 473, 473, generator=g) < 0.1) & (gt == 0)).long() if with_ignore else None
    padded = F.pad(gt, (0, 7, 0, 7), value=-1).cuda()
    pad_ignore = F.pad(ignore, (0, 7, 0, 7), value=0).cuda() if with_ignore else None
    meter = FewShotMeter(20, [3, 7, 19])
    zs.update_metric(meter, x, class_info.cuda(), padded, pad_ignore)
    want = rule_counts(mask.cpu().numpy(), fewshot_target(gt.numpy(), None if ignore is None else ignore.numpy()), 2,
                       class_info.numpy(), 20)
    assert np.array_equal(meter.stats.cpu().numpy(), want)
    # the same through classify_prediction + update on the cropped mask
    meter2 = FewShotMeter(20, [3, 7, 19])
    inter, union = classify_prediction(mask, gt.cuda(), None if ignore is None else ignore.cuda())
    meter2.update(inter, union, class_info.cuda())
    assert torch.equal(meter2.intersection_buf, meter.intersection_buf)
    assert torch.equal(meter2.union_buf, meter.union_buf)
    _no_error(ops)


def test_segmentation_metric_sequence(ops):
    """lists, [H,W] targets, CPU targets, fp16 scores and masks, against the encoding restatement"""
    from lseg_b200.metrics import SegmentationMetric, batch_intersection_union, batch_pix_accuracy
    nclass = 150
    g = torch.Generator().manual_seed(3)
    metric = SegmentationMetric(nclass)
    ref = EncodingMetric(nclass)
    for step in range(4):
        s = torch.randn(1, nclass, 37, 41, generator=g)
        p = s.argmax(1)
        t = _targets(g, (1, 37, 41), nclass, p)
        if step == 0:
            metric.update(t[0], s.cuda())                      # [H,W] CPU target
        elif step == 1:
            metric.update([t[0].cuda(), t[0]], [s.cuda(), s.cuda()])  # list input
            ref.update(t[0].numpy(), p.numpy())
        elif step == 2:
            metric.update(t.cuda(), s.half().float().cuda().half())  # fp16 scores
            p = s.half().float().argmax(1)
        else:
            metric.update(t.cuda(), p.cuda())                  # int64 mask
        ref.update(t.numpy(), p.numpy())
        c, lab = batch_pix_accuracy(s.cuda(), t.cuda())
        assert (c, lab) == tuple(split(rule_counts(s.argmax(1).numpy(), t.numpy(), nclass)[0], nclass)[2:])
        inter, union = batch_intersection_union(s.cuda(), t.cuda(), nclass)
        want = split(rule_counts(s.argmax(1).numpy(), t.numpy(), nclass)[0], nclass)
        assert np.array_equal(inter, want[0]) and np.array_equal(union, want[1])
    got_all, want_all = metric.get_all(), ref.get_all()
    assert got_all[0] == want_all[0] and got_all[1] == want_all[1]
    assert np.array_equal(got_all[2], want_all[2]) and np.array_equal(got_all[3], want_all[3])
    assert metric.get() == ref.get()
    metric.reset()
    assert metric.get_all()[1] == 0


def test_fewshot_reproduces_reference_golden(ops):
    import os
    from lseg_b200.metrics import FewShotMeter, classify_prediction
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_metrics_fss.npz"))
    meter = FewShotMeter(int(gold["n_classes"]), gold["class_ids"])
    for i in range(gold["pred"].shape[0]):
        pred = torch.from_numpy(gold["pred"][i].astype(np.int64)).cuda()
        gt = torch.from_numpy(gold["gt"][i].astype(np.int64)).cuda()
        ignore = torch.from_numpy(gold["ignore"][i].astype(np.int64)).cuda() if gold["has_ignore"][i] else None
        keep = (pred.clone(), gt.clone(), None if ignore is None else ignore.clone())
        inter, union = classify_prediction(pred, gt, ignore)
        assert np.array_equal(inter.cpu().numpy(), gold["area_inter"][i])
        assert np.array_equal(union.cpu().numpy(), gold["area_union"][i])
        assert torch.equal(pred, keep[0]) and torch.equal(gt, keep[1])  # inputs left unchanged
        assert ignore is None or torch.equal(ignore, keep[2])
        meter.update(inter, union, torch.from_numpy(gold["class_id"][i]).cuda())
    assert np.array_equal(meter.intersection_buf.cpu().numpy(), gold["intersection_buf"])
    assert np.array_equal(meter.union_buf.cpu().numpy(), gold["union_buf"])
    miou, fb_iou = meter.compute_iou()
    want = fewshot_iou(gold["intersection_buf"], gold["union_buf"], gold["class_ids"])
    assert miou.item() == pytest.approx(want[0], rel=1e-12) and fb_iou.item() == pytest.approx(want[1], rel=1e-12)
    assert miou.item() == pytest.approx(float(gold["miou"]), rel=1e-6)
    assert fb_iou.item() == pytest.approx(float(gold["fb_iou"]), rel=1e-6)


def test_no_host_sync(ops, net, zs):
    from lseg_b200.metrics import FewShotMeter, SegmentationMetric
    tokens = synth.tokenize(synth.ade20k_labels()[:10])
    x = synth.make_image(2, 64, 96, seed=1).cuda()
    target = torch.randint(-1, 10, (2, 64, 96), device="cuda")
    scores = torch.randn(1, 10, 33, 35, device="cuda")
    t1 = torch.randint(-1, 10, (33, 35), device="cuda")
    metric = SegmentationMetric(10, device="cuda")
    net.update_metric(metric, x, target, tokens)  # warm: plans and text features
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        metric.update(t1, scores)
        metric.update([t1], [scores])
        net.update_metric(metric, x, target, tokens)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the zero-shot path keeps forward()'s host-side class_info range check and nothing else
    meter = FewShotMeter(20, [1, 2])
    ci = torch.tensor([1, 2], device="cuda")
    zs.update_metric(meter, x, ci, target.clamp(max=1))
    torch.cuda.synchronize()
    from unittest import mock
    text = zs._image_text(zs._engine_for(x.device), ci, x.device)
    torch.cuda.synchronize()
    with mock.patch.object(zs, "_image_text", lambda eng, c, d: text):
        torch.cuda.set_sync_debug_mode("error")
        try:
            zs.update_metric(meter, x, ci, target.clamp(max=1))
        finally:
            torch.cuda.set_sync_debug_mode(0)
    _no_error(ops)


def test_update_metric_rejects_bad_arguments(ops, net):
    from lseg_b200.metrics import SegmentationMetric
    eng = net._engine_for(torch.device("cuda"))
    tokens = synth.tokenize(synth.ade20k_labels()[:4])
    feats = net._text_features(eng, tokens)
    x = synth.make_image(1, 64, 64, seed=0).cuda()
    t = torch.zeros(1, 64, 64, dtype=torch.int64, device="cuda")
    s = torch.zeros(1, row_len(4), dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="target"):
        eng.forward_stats(x, feats, 4, t[:, :32], s, 4)
    with pytest.raises(ValueError, match="stats"):
        eng.forward_stats(x, feats, 4, t, s[:, :-1], 4)
    from lseg_b200._lib import LsegError
    x_wide = synth.make_image(1, 32, 1056, seed=0).cuda()
    with pytest.raises(LsegError, match="W <= 1024"):
        eng.forward_stats(x_wide, feats, 4, torch.zeros(1, 32, 1056, dtype=torch.int64, device="cuda"), s, 4)
    with pytest.raises(ValueError, match="CUDA"):
        SegmentationMetric(4).update(t.cpu(), torch.zeros(1, 4, 64, 64))
    assert not s.any()


@pytest.mark.parametrize("with_mask", [False, True])
def test_fused_out_of_range_group(ops, net, with_mask):
    """The fused output stage skips an image whose group id is outside [0, G) and reports it (tag 78); a requested mask
    is still written in full and equals predict()."""
    K, nclass = 6, 6
    tokens = synth.tokenize(synth.ade20k_labels()[:K])
    x = synth.make_image(3, 64, 96, seed=31).cuda()
    eng = net._engine_for(x.device)
    feats = net._text_features(eng, tokens)
    ref_mask = net.predict(x, tokens)
    g = torch.Generator().manual_seed(31)
    target = _targets(g, (3, 64, 96), nclass, ref_mask).cuda()
    group = torch.tensor([1, 7, 0], dtype=torch.int32)
    stats = torch.zeros((2, row_len(nclass)), dtype=torch.int64, device="cuda")
    mask = torch.full_like(ref_mask, -7) if with_mask else None
    _no_error(ops)
    eng.forward_stats(x, feats, K, target, stats, nclass, group=group.cuda(), mask=mask)
    wd = ops.read_watchdog()
    assert wd == [78, 1, 7, 2], wd
    want = rule_counts(ref_mask.cpu().numpy(), target.cpu().numpy(), nclass, group.numpy(), 2)
    assert np.array_equal(stats.cpu().numpy(), want)
    if with_mask:
        assert torch.equal(mask, ref_mask)


def test_fewshot_meter_raises_on_skipped_image(ops, zs):
    """class_info inside the label list but beyond the meter's rows: the image is not counted and compute_iou() says so
    (the reference's index_add_ fails on such a class id)."""
    from lseg_b200.metrics import FewShotMeter
    meter = FewShotMeter(10, [1, 2, 3])
    x = synth.make_image(2, 64, 96, seed=5).cuda()
    target = torch.randint(0, 2, (2, 64, 96), device="cuda")
    zs.update_metric(meter, x, torch.tensor([3, 15], device="cuda"), target)
    with pytest.raises(RuntimeError, match=r"skipped image 1 of its batch: its row id 15 is outside \[0, 10\)"):
        meter.compute_iou()
    mask = zs.predict(x, torch.tensor([3, 15], device="cuda"))
    want = rule_counts(mask.cpu().numpy(), target.cpu().numpy(), 2, [3, 15], 10)
    assert np.array_equal(meter.stats.cpu().numpy(), want)
    meter.compute_iou()  # the record was consumed by the first read
