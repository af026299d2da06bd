"""GPU tests of encode-once / query-many (LSegNet.encode_image, PixelEmbedding, lseg_query) and of the embedding export
(lseg_embedding_features): a query returns what the forward of the encoded images returns, bit for bit, on every net
and output kind; embeddings survive other work on the engine; batches slice and concatenate; the exported features
match float64, the oracle and the reference; a query allocates only the tail's buffers; bad arguments are rejected by
name; the multi-scale evaluator replays stored embeddings bit for bit."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import embed_oracle as E
from parity_util import NET_KW, oracle_forward, rel_err, state_dict, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
STAGE_TOL = 1.0e-3  # fp32 stages of the oracle vs the engine (tests/test_model_gpu.py)


@pytest.fixture(scope="module")
def net():
    import lseg_b200  # noqa: F401
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


def _labels(k):
    if k <= 150:
        return synth.tokenize(synth.ade20k_labels()[:k])
    return synth.synthetic_prompts(k, seed=0)


def _assert_same_outputs(net, x, emb, tokens, nclass):
    """forward / predict / update_metric on the embedding vs on the images: equal bit for bit."""
    from lseg_b200.metrics import SegmentationMetric
    assert torch.equal(net(emb, tokens), net(x, tokens))
    assert torch.equal(net.predict(emb, tokens), net.predict(x, tokens))
    target = torch.randint(-1, nclass, (x.shape[0], x.shape[2], x.shape[3]), generator=torch.Generator().manual_seed(1))
    m_x, m_e = SegmentationMetric(nclass), SegmentationMetric(nclass)
    net.update_metric(m_x, x, target.cuda(), tokens)
    net.update_metric(m_e, emb, target.cuda(), tokens)
    assert torch.equal(m_x.stats, m_e.stats) and int(m_x.stats.sum()) > 0


# ------------------------------------------------------------------------------------------------
# 1. bit identity with the existing calls
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,K", [(2, 64, 96, 5), (1, 480, 480, 150), (8, 480, 480, 150), (2, 160, 224, 7),
                                     (1, 736, 736, 512)])
def test_query_equals_forward(net, B, H, W, K):
    tokens = _labels(K)
    x = synth.make_image(B, H, W, seed=B * 1000 + H).cuda()
    emb = net.encode_image(x)
    assert emb.emb.shape == (B, H // 2, W // 2, 512) and emb.emb.dtype == torch.float16
    assert emb.sumsq.shape == (B, H // 2, W // 2, 16) and emb.sumsq.dtype == torch.float32
    _assert_same_outputs(net, x, emb, tokens, min(K, 150))
    out = torch.full((B, K, H, W), float("nan"), device="cuda")
    assert net(emb, tokens, out=out) is out and torch.equal(out, net(x, tokens))


@pytest.mark.parametrize("tag,kw", [("opt1", dict(arch_option=1, block_depth=2, activation="lrelu")),
                                    ("opt2", dict(arch_option=2, block_depth=3, activation="tanh"))])
def test_query_equals_forward_arch_option(tag, kw):
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels()[:5], **{**NET_KW, **kw})
    n.load_state_dict(synth.make_state_dict(0, head_block=True))
    n = n.cuda().eval()
    x = synth.make_image(2, 64, 96, seed=2064).cuda()
    _assert_same_outputs(n, x, n.encode_image(x), synth.tokenize(synth.ade20k_labels()[:5]), 5)


@pytest.mark.parametrize("backbone", ["clip_vitb32_384", "clipRN50x16_vitl16_384"])
def test_query_equals_forward_other_backbones(backbone):
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels(), **{**NET_KW, "backbone": backbone})
    n.load_state_dict(state_dict(0, backbone))
    n = n.cuda().eval()
    tokens = synth.tokenize(synth.ade20k_labels()[:7])
    for B, H, W in ((3, 160, 224), (2, 480, 480)):
        x = synth.make_image(B, H, W, seed=H).cuda()
        emb = n.encode_image(x)
        assert emb.out_c == n.out_c and emb.emb.shape[3] == n.out_c
        _assert_same_outputs(n, x, emb, tokens, 7)
        f = emb.features()
        assert f.shape == (B, n.out_c, H // 2, W // 2)
        assert (f.double().norm(dim=1) - 1).abs().max().item() < 1e-3  # unit rows up to the fp16 storage of emb


@pytest.mark.parametrize("kind", ["vit", "rn101"])
def test_zero_shot_query_equals_forward(kind):
    from lseg_b200.lseg_net import LSegNetZS, LSegRNNetZS
    from lseg_b200.metrics import FewShotMeter
    names = [f"class {i}" for i in range(20)]
    if kind == "vit":
        n = LSegNetZS(label_list=names, **NET_KW)
        n.load_state_dict(state_dict(0))
    else:
        n = LSegRNNetZS(label_list=names, features=256, arch_option=0, block_depth=0, activation="lrelu")
        n.load_state_dict(state_dict(0, "clip_resnet101"))
    n = n.cuda().eval()
    x = synth.make_image(4, 96, 128, seed=5).cuda()
    class_info = torch.tensor([3, 7, 3, 19])
    emb = n.encode_image(x)
    assert torch.equal(n(emb, class_info), n(x, class_info))
    assert torch.equal(n.predict(emb, class_info), n.predict(x, class_info))
    target = torch.randint(-1, 2, (4, 96, 128), generator=torch.Generator().manual_seed(2)).cuda()
    m_x, m_e = FewShotMeter(20, [3, 7, 19]), FewShotMeter(20, [3, 7, 19])
    n.update_metric(m_x, x, class_info.cuda(), target)
    n.update_metric(m_e, emb, class_info.cuda(), target)
    assert torch.equal(m_x.stats, m_e.stats) and int(m_x.stats.sum()) > 0


# ------------------------------------------------------------------------------------------------
# 2. persistence: the engine keeps no reference to a stored embedding
# ------------------------------------------------------------------------------------------------
def test_embedding_survives_other_work(net):
    tokens = _labels(5)
    x = synth.make_image(2, 160, 224, seed=1).cuda()
    emb = net.encode_image(x)
    before = net(emb, tokens)
    mask_before = net.predict(emb, tokens)
    net(synth.make_image(2, 160, 224, seed=2).cuda(), tokens)  # same shape: overwrites the plan's own embedding
    net.encode_image(synth.make_image(2, 160, 224, seed=3).cuda())
    for B, H, W in ((1, 64, 64), (3, 96, 96), (2, 128, 64), (1, 64, 128)):  # more shapes than the plan / tail caches hold
        net(synth.make_image(B, H, W, seed=H + W).cuda(), tokens)
        net(net.encode_image(synth.make_image(B, H, W, seed=H).cuda()), _labels(7))
    assert torch.equal(net(emb, tokens), before)
    assert torch.equal(net.predict(emb, tokens), mask_before)


# ------------------------------------------------------------------------------------------------
# 3. batch algebra (deterministic mode: batch-invariant, tests/test_model_gpu.py::test_batch_consistency)
# ------------------------------------------------------------------------------------------------
def test_slices_and_concatenation(net):
    from lseg_b200 import ops
    from lseg_b200.lseg_net import PixelEmbedding
    tokens = _labels(5)
    x = synth.make_image(8, 480, 480, seed=5).cuda()
    ops.set_deterministic(True)
    emb = net.encode_image(x)
    full = net(emb, tokens)
    full_mask = net.predict(emb, tokens)
    for i, j in ((0, 3), (3, 8), (5, 6)):
        assert len(emb[i:j]) == j - i
        assert torch.equal(net(emb[i:j], tokens), full[i:j])
        assert torch.equal(net.predict(emb[i:j], tokens), full_mask[i:j])
    cat = PixelEmbedding.cat([net.encode_image(x[:3]), net.encode_image(x[3:])])
    assert torch.equal(cat.emb, emb.emb) and torch.equal(cat.sumsq, emb.sumsq)
    assert torch.equal(net(cat, tokens), full)


# ------------------------------------------------------------------------------------------------
# 4. features(): float64, oracle, reference
# ------------------------------------------------------------------------------------------------
def _feature_bound(C):
    """Relative error of emb * rsqrt(sum of the C/32 fp32 partials) against the float64 normalisation of the same stored
    fp16 rows and fp32 partials, u = 2^-24 (fp32 unit roundoff):
      sequential fp32 sum of n = C/32 positive terms     |rel| <= (n - 1) u   -> through rsqrt: (n - 1) u / 2
      rsqrtf (CUDA C Programming Guide: 2 ulp)           |rel| <= 2 * 2u
      the product x * r rounded to fp32                  |rel| <= u
    plus 1 % for second-order terms."""
    u = 2.0 ** -24
    n = C // 32
    return 1.01 * ((n - 1) * u / 2 + 4 * u + u)


def test_features_against_float64(net):
    for B, H, W in ((2, 64, 96), (1, 480, 480)):
        emb = net.encode_image(synth.make_image(B, H, W, seed=7).cuda())
        f = emb.features()
        assert f.shape == (B, 512, H // 2, W // 2) and f.dtype == torch.float32 and f.is_contiguous()
        e64 = emb.emb.double()
        s64 = emb.sumsq.double().sum(-1, keepdim=True)
        ref = (e64 / s64.sqrt()).permute(0, 3, 1, 2)
        err = (f.double() - ref).abs()
        bound = _feature_bound(512) * ref.abs()
        assert bool((err <= bound).all()), (err - bound).max().item()


@pytest.mark.parametrize("B,H,W", [(2, 64, 96), (1, 480, 480)])
def test_features_against_oracle_and_reference(net, B, H, W):
    seed = {64: 2064, 480: 1480}[H]
    x = synth.make_image(B, H, W, seed=seed)
    _, st = oracle_forward(x, synth.tokenize(["cat", "other"]))
    ref = E.image_features(st["path_1"], state_dict(0))
    f = net.encode_image(x.cuda()).features().cpu()
    # stored in fp16 (emb): the stage tolerance + one fp16 quantum of the largest component
    mx = ref.abs().max().item()
    tol = STAGE_TOL + 2.0 ** (math.floor(math.log2(mx)) - 10) / mx
    assert rel_err(f, ref) <= tol, rel_err(f, ref)
    z = np.load(os.path.join(GOLD, "ref_embed.npz"))
    tag = "small" if H == 64 else "s480"
    s = int(z[f"{tag}_stride"])
    assert rel_err(f[:, :, ::s, ::s], torch.from_numpy(z[tag])) <= tol


def test_features_768_channels():
    """C = 768 (RN50x16 text width) through the ABI entry directly."""
    from lseg_b200.engine import embedding_features
    g = torch.Generator(device="cuda").manual_seed(3)
    emb = torch.randn((2, 16, 32, 768), generator=g, device="cuda").half()  # the grid of a 32x64 image
    sumsq = emb.float().pow(2).view(2, 16, 32, 24, 32).sum(-1).contiguous()
    f = embedding_features(emb, sumsq)
    ref = (emb.double() / sumsq.double().sum(-1, keepdim=True).sqrt()).permute(0, 3, 1, 2)
    assert bool(((f.double() - ref).abs() <= _feature_bound(768) * ref.abs()).all())


# ------------------------------------------------------------------------------------------------
# 5. memory: a query allocates the tail's buffers, not the trunk's arena
# ------------------------------------------------------------------------------------------------
def test_query_without_trunk_plan_allocates_only_the_tail(net):
    B, H, W, K = 2, 224, 160, 9
    tokens = _labels(K)
    emb = net.encode_image(synth.make_image(B, H, W, seed=9).cuda())
    for h, w in ((64, 64), (96, 96), (64, 128), (128, 64)):  # evict the (B, H, W) plan and tail
        net(synth.make_image(B, h, w, seed=h).cuda(), tokens)
    out = torch.empty((B, K, H, W), device="cuda")
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    net(emb, tokens, out=out)
    torch.cuda.synchronize()
    grown = free0 - torch.cuda.mem_get_info()[0]
    tail = B * K * (H // 2) * (W // 2) * 2  # fp16 low-res logits
    slack = 8 << 20  # cudaMalloc granularity (2 MB pages) and driver bookkeeping
    assert grown <= tail + slack, (grown, tail)


# ------------------------------------------------------------------------------------------------
# 6. errors
# ------------------------------------------------------------------------------------------------
def test_python_rejects_bad_embeddings(net):
    from lseg_b200.lseg_net import LSegNet
    tokens = _labels(3)
    emb = net.encode_image(synth.make_image(1, 64, 64, seed=1).cuda())
    eng = net._engine_for(torch.device("cuda"))
    text = net._text_features(eng, tokens)
    out = torch.empty((1, 3, 64, 64), device="cuda")
    cases = [
        ("emb", dict(emb=emb.emb.float())),                                  # dtype
        ("emb", dict(emb=emb.emb[:, :, :, :256].contiguous())),              # channels
        ("sumsq", dict(sumsq=emb.sumsq[:, :, :, :8].contiguous())),          # shape
        ("embedding is on", dict(emb=emb.emb.cpu(), sumsq=emb.sumsq.cpu())),  # device
        ("logits", dict(logits=torch.empty((1, 3, 64, 32), device="cuda"))),
        ("no output", dict(logits=None)),
        ("target and stats", dict(target=torch.zeros((1, 64, 64), dtype=torch.int64, device="cuda"))),
    ]
    for msg, kw in cases:
        args = dict(emb=emb.emb, sumsq=emb.sumsq, logits=out)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            eng.query(args.pop("emb"), args.pop("sumsq"), text, 3, **args)
    other = LSegNet(labels=["a"], **{**NET_KW, "backbone": "clip_vitb32_384"})
    with pytest.raises(ValueError, match="backbone"):
        other.cuda().eval()(emb, tokens)
    net.refresh()  # weights may have changed: stored embeddings are stale
    with pytest.raises(ValueError, match="weights"):
        net(emb, tokens)
    with pytest.raises(ValueError, match="weights"):
        net.predict(emb, tokens)


def test_abi_rejects_bad_arguments_before_launching(net):
    from lseg_b200 import _lib
    lib = _lib.load()
    eng = net._engine_for(torch.device("cuda"))
    emb, sumsq = eng.encode_image(synth.make_image(1, 64, 64, seed=1).cuda())
    text = net._text_features(eng, _labels(3))
    mask = torch.full((1, 64, 64), -7, dtype=torch.int64, device="cuda")
    target = torch.zeros((1, 64, 64), dtype=torch.int64, device="cuda")
    stats = torch.zeros((1, 3 * 3 + 2), dtype=torch.int64, device="cuda")
    P = C.c_void_p
    good = dict(e=eng.handle, emb=P(emb.data_ptr()), sumsq=P(sumsq.data_ptr()), B=1, H=64, W=64, text=P(text.data_ptr()),
                K=3, stride=0, logits=None, mask=P(mask.data_ptr()), target=None, group=None, nclass=0, G=0, stats=None)
    wide = torch.zeros((1, 64, 2048), dtype=torch.int64, device="cuda")
    cases = [
        ("null emb", dict(emb=None)), ("null emb_sumsq", dict(sumsq=None)), ("null text", dict(text=None)),
        ("emb must be 16-byte aligned", dict(emb=P(emb.data_ptr() + 2))),
        ("mask must be 8-byte aligned", dict(mask=P(mask.data_ptr() + 4))),
        ("multiples of 32", dict(H=48)), ("multiples of 32", dict(W=80)), ("B=0", dict(B=0)),
        ("K=0", dict(K=0)), ("text_image_stride", dict(stride=2)),
        ("no output", dict(mask=None)),
        ("null target", dict(stats=P(stats.data_ptr()), nclass=3, G=1)),
        ("nclass", dict(target=P(target.data_ptr()), stats=P(stats.data_ptr()), nclass=0, G=1)),
        ("W=2048", dict(target=P(wide.data_ptr()), stats=P(stats.data_ptr()), nclass=3, G=1, W=2048)),
    ]
    for msg, kw in cases:
        a = dict(good)
        a.update(kw)
        rc = lib.lseg_query(a["e"], a["emb"], a["sumsq"], a["B"], a["H"], a["W"], a["text"], a["K"], a["stride"],
                            a["logits"], a["mask"], a["target"], a["group"], a["nclass"], a["G"], a["stats"], None)
        err = lib.lseg_last_error().decode()
        assert rc != 0 and msg in err, (msg, err)
    torch.cuda.synchronize()
    assert bool((mask == -7).all()) and int(stats.abs().sum()) == 0  # nothing ran
    with pytest.raises(_lib.LsegError, match="C=640"):
        _lib.check(lib.lseg_embedding_features(P(emb.data_ptr()), P(sumsq.data_ptr()), 1, 32, 32, 640,
                                               P(mask.data_ptr()), None))
    with pytest.raises(_lib.LsegError, match="null emb"):
        _lib.check(lib.lseg_encode_image(eng.handle, P(target.data_ptr()), 1, 64, 64, None, P(sumsq.data_ptr()), None))
    # the good call still works and writes the forward's mask
    rc = lib.lseg_query(*[good[k] for k in ("e", "emb", "sumsq", "B", "H", "W", "text", "K", "stride", "logits", "mask",
                                             "target", "group", "nclass", "G", "stats")], None)
    assert rc == 0
    assert torch.equal(mask, net.predict(synth.make_image(1, 64, 64, seed=1).cuda(), _labels(3)))


# ------------------------------------------------------------------------------------------------
# 7. the multi-scale evaluator on stored embeddings
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,base,crop,scales", [(50, 60, 64, 64, (0.5, 0.75, 1.0)),      # whole-image scales only
                                                  (90, 120, 96, 64, (0.75, 1.0, 1.5))])   # sliding windows
def test_evaluator_replays_embeddings(net, h, w, base, crop, scales):
    from lseg_b200.evaluator import MultiScaleEvaluator
    ev = MultiScaleEvaluator(net, base_size=base, crop_size=crop, scales=scales, max_batch=4)
    img = synth.make_image(1, h, w, seed=h).cuda()
    enc = ev.encode(img)
    assert len(enc.batches) == math.ceil(ev.num_forwards(img)[1] / 4)
    for labels in (["cat", "other", "tree"], synth.ade20k_labels()[:11]):
        assert torch.equal(ev(enc, labels), ev(img, labels))
        assert torch.equal(ev.predict(enc, labels), ev.predict(img, labels))
    with pytest.raises(TypeError):
        MultiScaleEvaluator(net, base_size=base, crop_size=crop, scales=scales, fused=False).encode(img)
    with pytest.raises(TypeError):
        MultiScaleEvaluator(lambda x, l: x, base_size=base, crop_size=crop, scales=scales).encode(img)
