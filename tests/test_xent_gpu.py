"""GPU checks of the device cross-entropy (csrc/xent.cuh, the loss variant of the fused output stage): every loss is fed
the engine's own logits (forward's output) and compared against the float64 oracle of tests/xent_oracle.py within the
derived bound of the kernel's fp32 sequence, and against torch's CUDA F.cross_entropy within twice that bound."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity_util import NET_KW, state_dict, synth
from segstats_oracle import row_len
from xent_oracle import mean_bound, xent_mean

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops
    ops.read_watchdog()  # start from a clear error record
    return ops


def _no_error(ops):
    wd = ops.read_watchdog()
    assert wd[0] == 0, f"watchdog / metric / loss error record set: {wd}"


def _target(seed, B, H, W, K, ignore_index=-1, frac=0.2):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, K, (B, H, W), generator=g)
    t = torch.where(torch.rand(B, H, W, generator=g) < frac, torch.full_like(t, ignore_index), t)
    return t.cuda()


def _check(loss, logits, target, ignore_index=-1):
    """loss (the device's) within the bound of the float64 oracle, and torch's CUDA cross-entropy within twice it."""
    lg, t = logits.cpu().numpy(), target.cpu().numpy()
    want = xent_mean(lg, t, ignore_index)
    bound = mean_bound(lg, t, ignore_index)
    got = loss.item()
    assert loss.dtype == torch.float32 and loss.dim() == 0 and loss.is_cuda
    assert abs(got - want) <= bound, (got, want, bound)
    ref = F.cross_entropy(logits, target, ignore_index=ignore_index).item()
    assert abs(got - ref) <= 2 * bound, (got, ref, bound)
    return bound


_NETS = {}


def _net(kind):
    if kind in _NETS:
        return _NETS[kind]
    from lseg_b200.lseg_net import LSegNet, LSegNetZS, LSegRNNetZS
    names = [f"class {i}" for i in range(20)]
    if kind == "vitl16":
        n = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
        n.load_state_dict(state_dict(0))
    elif kind == "vitb32":
        n = LSegNet(labels=synth.ade20k_labels(), **{**NET_KW, "backbone": "clip_vitb32_384"})
        n.load_state_dict(state_dict(0, "clip_vitb32_384"))
    elif kind in ("opt1", "opt2"):
        kw = dict(arch_option=1, block_depth=2, activation="lrelu") if kind == "opt1" else \
            dict(arch_option=2, block_depth=3, activation="tanh")
        n = LSegNet(labels=synth.ade20k_labels(), **{**NET_KW, **kw})
        n.load_state_dict(synth.make_state_dict(0, head_block=True))
    elif kind == "zs":
        n = LSegNetZS(label_list=names, **NET_KW)
        n.load_state_dict(state_dict(0))
    else:
        n = LSegRNNetZS(label_list=names, features=256, arch_option=0, block_depth=0, activation="lrelu")
        n.load_state_dict(state_dict(0, "clip_resnet101"))
    _NETS[kind] = n.cuda().eval()
    return _NETS[kind]


def _labels(K):
    return synth.tokenize(synth.ade20k_labels()[:K] if K <= 150 else [f"label {i}" for i in range(K)])


CASES = [  # (net, B, H, W, K, ignore_index)
    ("vitl16", 1, 32, 32, 1, -1),
    ("vitl16", 1, 32, 480, 2, -1),
    ("vitl16", 8, 32, 1024, 150, -1),
    ("vitl16", 1, 32, 480, 1365, 255),
    ("vitl16", 8, 32, 480, 150, 255),
    ("vitb32", 2, 64, 96, 150, -1),
    ("opt1", 2, 32, 480, 150, -1),
    ("opt2", 1, 32, 1024, 150, -1),
]


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}_B{c[1]}_{c[2]}x{c[3]}_K{c[4]}_i{c[5]}" for c in CASES])
def test_fused_loss_against_oracle(ops, case):
    kind, B, H, W, K, ign = case
    net = _net(kind)
    x = synth.make_image(B, H, W, seed=H + W + K).cuda()
    tokens = _labels(K)
    logits = net(x, tokens)
    target = _target(B + K, B, H, W, K, ign)
    loss = net.loss(x, target, tokens, ignore_index=ign)
    if K == 1:
        assert loss.item() == 0.0
    _check(loss, logits, target, ign)
    # the standalone scores op on the same logits agrees within the same bound
    from lseg_b200.metrics import SegmentationLosses
    alone = SegmentationLosses(ignore_index=ign)(logits, target)
    _check(alone, logits, target, ign)
    assert abs(alone.item() - loss.item()) <= 2 * mean_bound(logits.cpu().numpy(), target.cpu().numpy(), ign)
    _no_error(ops)


@pytest.mark.parametrize("kind", ["zs", "rn"])
def test_zero_shot_loss_and_meter(ops, kind):
    """The per-image ['others', name] pairs: loss over the raw target; with a meter, its counters equal
    update_metric's and loss_buf gets the loss."""
    from lseg_b200.metrics import FewShotMeter
    net = _net(kind)
    B, H, W = 4, 96, 128
    x = synth.make_image(B, H, W, seed=31).cuda()
    ci = torch.tensor([3, 0, 7, 3])
    target = _target(5, B, H, W, 2, -1)
    qi = (torch.rand(B, H, W, generator=torch.Generator().manual_seed(2)) < 0.1).long().cuda()
    logits = net(x, ci)
    m1, m2 = FewShotMeter(20, list(range(20))), FewShotMeter(20, list(range(20)))
    loss = net.loss(x, ci, target, meter=m1, query_ignore_idx=qi)
    net.update_metric(m2, x, ci, target, query_ignore_idx=qi)
    assert torch.equal(m1.stats, m2.stats)
    assert len(m1.loss_buf) == 1 and torch.equal(m1.loss_buf[0], loss)
    _check(loss, logits, target)
    assert torch.equal(net.loss(x, ci, target), loss)
    _no_error(ops)


def test_loss_with_metric_one_call(ops):
    """Loss + counters + mask + logits in one launch: counters == update_metric's, mask == predict, logits == forward,
    loss bits == the loss-only call's; the same call twice gives the same bits; an embedding gives the same bits."""
    from lseg_b200.metrics import SegmentationMetric
    net = _net("vitl16")
    B, H, W, K = 2, 256, 384, 150
    x = synth.make_image(B, H, W, seed=3).cuda()
    tokens = _labels(K)
    target = _target(9, B, H, W, K, -1)
    m_ref = SegmentationMetric(K)
    net.update_metric(m_ref, x, target, tokens)
    m = SegmentationMetric(K)
    loss = net.loss(x, target, tokens, metric=m)
    assert torch.equal(m.stats, m_ref.stats)
    loss_only = net.loss(x, target, tokens)
    assert torch.equal(loss, loss_only)
    assert torch.equal(net.loss(x, target, tokens), loss_only)  # deterministic
    eng = net._engine_for(x.device)
    feats = net._text_features(eng, tokens)
    acc = torch.zeros(2, dtype=torch.float64, device="cuda")
    stats = torch.zeros((1, row_len(K)), dtype=torch.int64, device="cuda")
    mask = torch.full((B, H, W), -7, dtype=torch.int64, device="cuda")
    logits = torch.empty((B, K, H, W), device="cuda")
    eng.forward_loss(x, feats, K, target, acc, target=target, stats=stats, nclass=K, mask=mask, logits=logits)
    assert torch.equal(stats, m_ref.stats)
    assert torch.equal(mask, net.predict(x, tokens))
    assert torch.equal(logits, net(x, tokens))
    assert torch.equal((acc[0] / acc[1]).float(), loss)
    emb = net.encode_image(x)
    assert torch.equal(net.loss(emb, target, tokens), loss)
    m_emb = SegmentationMetric(K)
    assert torch.equal(net.loss(emb, target, tokens, metric=m_emb), loss)
    assert torch.equal(m_emb.stats, m_ref.stats)
    _check(loss, logits, target)
    with pytest.raises(ValueError, match="per-image"):
        net.loss(x, target, [["a"], ["b"]])
    _no_error(ops)


def test_all_ignored_is_nan(ops):
    net = _net("vitl16")
    x = synth.make_image(1, 32, 64, seed=1).cuda()
    t = torch.full((1, 32, 64), 255, dtype=torch.int64, device="cuda")
    assert torch.isnan(net.loss(x, t, _labels(5), ignore_index=255))
    from lseg_b200.metrics import SegmentationLosses
    assert torch.isnan(SegmentationLosses(ignore_index=255)(net(x, _labels(5)), t))
    _no_error(ops)


@pytest.mark.parametrize("path", ["fused", "scores"])
def test_out_of_range_target_gives_nan_and_record(ops, path):
    from lseg_b200.metrics import SegmentationLosses, _raise_on_device_error
    net = _net("vitl16")
    B, H, W, K = 2, 32, 64, 5
    x = synth.make_image(B, H, W, seed=2).cuda()
    t = _target(3, B, H, W, K, -1)
    t[1, 3, 7] = K + 250
    if path == "fused":
        loss = net.loss(x, t, _labels(K))
    else:
        loss = SegmentationLosses()(net(x, _labels(K)), t)
    assert torch.isnan(loss)
    with pytest.raises(RuntimeError, match=r"target 255 at pixel 199 .* image 1 "):
        _raise_on_device_error(x.device)
    _no_error(ops)


@pytest.mark.parametrize("B,K,H,W", [(1, 150, 512, 683), (3, 2, 7, 9), (2, 1365, 33, 31), (1, 1, 5, 5)])
def test_scores_op_against_oracle(ops, B, K, H, W):
    """The standalone op at evaluator-like shapes (any H, W); fed logits of the engine's range (synthetic here: the op
    does not depend on where the scores come from)."""
    from lseg_b200.metrics import SegmentationLosses
    g = torch.Generator().manual_seed(B + K + H)
    scores = (torch.randn(B, K, H, W, generator=g) * 5).cuda()
    t = _target(K, B, H, W, K, -1)
    loss = SegmentationLosses()(scores, t)
    _check(loss, scores, t)
    assert torch.equal(SegmentationLosses()(scores, t), loss)
    if K == 1:
        assert loss.item() == 0.0
    _no_error(ops)


def test_rejects_bad_arguments_by_name(ops):
    """Every rejected argument is named before any launch, and the device error record stays clear."""
    from lseg_b200 import _lib
    lib = _lib.load()
    dev = torch.zeros(4096, dtype=torch.float64, device="cuda")
    p = C.c_void_p(dev.data_ptr())
    odd = C.c_void_p(dev.data_ptr() + 4)
    s = torch.cuda.current_stream().cuda_stream
    S = C.c_void_p(s)

    def scores(**kw):
        a = dict(scores=p, target=p, ign=-1, B=1, K=3, H=4, W=4, loss=p, part=p, n=64)
        a.update(kw)
        return lib.lseg_xent_scores(a["scores"], a["target"], a["ign"], a["B"], a["K"], a["H"], a["W"], a["loss"],
                                    a["part"], a["n"], S)

    for kw, msg in ((dict(scores=None), "null scores"), (dict(target=None), "null loss target"),
                    (dict(loss=None), "null loss accumulator"), (dict(part=None), "null partials"),
                    (dict(target=odd), "loss target must be 8-byte"), (dict(loss=odd), "accumulator must be 8-byte"),
                    (dict(part=odd), "partials must be 8-byte"), (dict(K=0), "K=0"), (dict(B=0), "B=0"),
                    (dict(B=70000), "B=70000"), (dict(H=0), "H=0"), (dict(n=1), "partials_len=1")):
        assert scores(**kw) != 0, kw
        assert msg in lib.lseg_last_error().decode(), (kw, lib.lseg_last_error())
    net = _net("vitl16")
    eng = net._engine_for(torch.device("cuda"))
    h = eng.handle

    def fwd(**kw):
        a = dict(e=h, x=p, B=1, H=32, W=32, text=p, K=2, target=None, group=None, stats=None, lt=p, loss=p, part=p,
                 n=64)
        a.update(kw)
        return lib.lseg_forward_xent(a["e"], a["x"], a["B"], a["H"], a["W"], a["text"], a["K"], 0, a["target"],
                                     a["group"], 1, 1, a["stats"], a["lt"], -1, a["loss"], a["part"], a["n"], None,
                                     None, S)

    for kw, msg in ((dict(e=None), "null engine"), (dict(x=None), "null x"), (dict(text=None), "null text"),
                    (dict(K=0), "K=0"), (dict(lt=None), "null loss target"), (dict(loss=None), "null loss accumulator"),
                    (dict(part=None), "null partials"), (dict(n=1), "partials_len=1"), (dict(W=1056), "W=1056"),
                    (dict(B=0), "B=0"), (dict(H=48), "H"), (dict(stats=p), "null target"),
                    (dict(target=p), "null stats"), (dict(loss=odd), "accumulator must be 8-byte")):
        assert fwd(**kw) != 0, kw
        assert msg in lib.lseg_last_error().decode(), (kw, lib.lseg_last_error())
    emb, sumsq = eng.encode_image(synth.make_image(1, 32, 32, seed=0).cuda())
    q = dict(e=h, emb=C.c_void_p(emb.data_ptr()), ss=C.c_void_p(sumsq.data_ptr()))

    def query(**kw):
        a = dict(q, text=p, K=2, lt=p, loss=p, part=p, n=64)
        a.update(kw)
        return lib.lseg_query_xent(a["e"], a["emb"], a["ss"], 1, 32, 32, a["text"], a["K"], 0, None, None, None, None,
                                   0, 0, None, a["lt"], -1, a["loss"], a["part"], a["n"], S)

    for kw, msg in ((dict(emb=None), "null emb"), (dict(ss=None), "null emb_sumsq"), (dict(text=None), "null text"),
                    (dict(K=0), "K=0"), (dict(lt=None), "null loss target"), (dict(n=3), "partials_len=3")):
        assert query(**kw) != 0, kw
        assert msg in lib.lseg_last_error().decode(), (kw, lib.lseg_last_error())
    torch.cuda.synchronize()
    assert not dev.any()  # nothing was launched on the buffers
    _no_error(ops)
