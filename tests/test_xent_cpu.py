"""CPU checks of the cross-entropy oracle (tests/xent_oracle.py) against torch, of its derived bound, and of the host-side
rules of lseg_b200.metrics.SegmentationLosses / FewShotMeter.loss_buf that need no device."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from xent_oracle import U, mean_bound, pixel_bound, rho, xent_mean


def _case(seed, B, K, H, W, ignore_index, frac_ignored=0.2):
    g = torch.Generator().manual_seed(seed)
    logits = (torch.randn(B, K, H, W, generator=g) * 4).float()
    t = torch.randint(0, K, (B, H, W), generator=g)
    t = torch.where(torch.rand(B, H, W, generator=g) < frac_ignored, torch.full_like(t, ignore_index), t)
    return logits, t


@pytest.mark.parametrize("ignore_index", [-1, 255])
@pytest.mark.parametrize("B,K,H,W", [(1, 1, 5, 7), (2, 2, 8, 8), (3, 150, 6, 9), (1, 1365, 3, 4)])
def test_oracle_equals_torch_float64(B, K, H, W, ignore_index):
    logits, t = _case(B * K + H, B, K, H, W, ignore_index)
    want = F.cross_entropy(logits.double(), t, ignore_index=ignore_index).item()
    got = xent_mean(logits.numpy(), t.numpy(), ignore_index)
    assert got == pytest.approx(want, rel=1e-12, abs=1e-12)


@pytest.mark.parametrize("ignore_index", [-1, 255])
def test_oracle_all_ignored_is_nan(ignore_index):
    logits, t = _case(1, 2, 4, 3, 3, ignore_index, frac_ignored=1.0)
    assert torch.isnan(F.cross_entropy(logits.double(), t, ignore_index=ignore_index))
    assert np.isnan(xent_mean(logits.numpy(), t.numpy(), ignore_index))


def test_oracle_out_of_range_target_is_nan():
    logits, t = _case(2, 1, 3, 4, 4, -1, frac_ignored=0.0)
    t[0, 1, 2] = 3
    assert np.isnan(xent_mean(logits.numpy(), t.numpy(), -1))


def test_bound_is_monotone_and_sane():
    ks = [1, 2, 150, 1365, 10 ** 5]
    r = [rho(k) for k in ks]
    assert all(a < b for a, b in zip(r, r[1:]))
    assert 0 < r[0] < 1e-6 and r[3] < 1e-3          # K = 1365: still far from 1
    assert r[3] > 1365 * 5 * U                       # at least the first-order term K (4u + u)
    base = pixel_bound(150, np.array(1.0), np.array(2.0), np.array(0.5))
    for kw in (dict(m=np.array(10.0)), dict(logS=np.array(5.0)), dict(vt=np.array(-30.0))):
        args = dict(m=np.array(1.0), logS=np.array(2.0), vt=np.array(0.5))
        args.update(kw)
        assert pixel_bound(150, **args) > base
    assert pixel_bound(2, np.array(1.0), np.array(2.0), np.array(0.5)) < base


def test_bound_covers_an_fp32_restatement():
    """The bound covers a plain fp32 evaluation of the same sequence (numpy float32, classes in order)."""
    logits, t = _case(5, 2, 150, 6, 6, -1)
    v = logits.numpy()
    m = np.full(t.shape, -np.inf, np.float32)
    s = np.zeros(t.shape, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for k in range(v.shape[1]):
            x = v[:, k]
            up = x > m
            s = np.where(up, s * np.exp(np.where(up, m - x, 0)).astype(np.float32) + np.float32(1),
                         s + np.exp(np.where(up, 0, x - m)).astype(np.float32)).astype(np.float32)
            m = np.maximum(m, x)
    counted = t.numpy() != -1
    vt = np.take_along_axis(v, np.where(counted, t.numpy(), 0)[:, None], 1)[:, 0]
    loss = ((m + np.log(s).astype(np.float32)).astype(np.float32) - vt).astype(np.float32)
    got = np.float32(loss[counted].astype(np.float64).mean())
    want = xent_mean(v, t.numpy(), -1)
    assert abs(float(got) - want) <= mean_bound(v, t.numpy(), -1)


def test_segmentation_losses_constructor_rules():
    from lseg_b200.metrics import SegmentationLosses
    c = SegmentationLosses(nclass=150, ignore_index=255)
    assert c.ignore_index == 255 and not c.se_loss and not c.aux
    for kw in (dict(se_loss=True), dict(aux=True), dict(weight=torch.ones(3))):
        with pytest.raises(NotImplementedError):
            SegmentationLosses(**kw)
    with pytest.raises(ValueError, match="CUDA"):
        c(torch.zeros(1, 2, 3, 3), torch.zeros(1, 3, 3, dtype=torch.int64))


def test_fewshot_meter_loss_buf_semantics():
    """AverageMeter.update appends the loss, torch.tensor(0.0) for None; reset empties the buffer. (CPU meter object
    built without its device buffers: only the loss bookkeeping is exercised.)"""
    from lseg_b200.metrics import FewShotMeter
    m = FewShotMeter.__new__(FewShotMeter)
    m.stats = torch.zeros((3, 8), dtype=torch.int64)
    m.loss_buf = []
    z = torch.zeros(2, 1, dtype=torch.int64)
    m.update(z, z, torch.tensor([1]), None)
    m.update(z, z, torch.tensor([2]), torch.tensor(0.75))
    assert [float(x) for x in m.loss_buf] == [0.0, 0.75]
    assert float(torch.stack(m.loss_buf).mean()) == pytest.approx(0.375)
    m.reset()
    assert m.loss_buf == []
