"""GPU tests of ragged batches — every image with its own label set (LSegNet.forward / predict with a list of label lists,
lseg_forward_ragged, lseg_query_ragged, lseg_gemm_ragged): each image's logits and mask equal a one-image call with its
own labels, bit for bit; equal label sets reduce to today's call; the embedding route gives the same bits; the engine
entry matches the per-image-block (text_image_stride) path; the GEMM stage op is exact on integer operands and writes
only its planes; cluster modes and arch_option 1 / 2 agree; bad arguments are rejected by name with outputs untouched."""
import ctypes as C

import pytest
import torch

from parity_util import NET_KW, state_dict, synth

pytestmark = pytest.mark.gpu

_POOL = synth.ade20k_labels() + [f"synthetic prompt {i}" for i in range(4000)]


def _sets(ks):
    """Disjoint label sets of the given sizes."""
    out, start = [], 0
    for k in ks:
        out.append(_POOL[start:start + k])
        start += k
    return out


@pytest.fixture(scope="module")
def net():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops
    from lseg_b200.lseg_net import LSegNet
    ops.set_deterministic(True)
    n = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


@pytest.fixture(scope="module")
def lib():
    from lseg_b200 import _lib
    return _lib.load()


def _check_per_image(net, x, sets, outs, mask):
    B, _, H, W = x.shape
    k = [len(s) for s in sets]
    assert isinstance(outs, list) and len(outs) == B
    assert mask.shape == (B, H, W) and mask.dtype == torch.int64
    base = outs[0].data_ptr()
    for b in range(B):
        assert outs[b].shape == (1, k[b], H, W) and outs[b].dtype == torch.float32
        assert outs[b].data_ptr() == base + 4 * sum(k[:b]) * H * W  # views of one packed buffer
        assert torch.equal(outs[b], net(x[b:b + 1], sets[b])), b
        assert torch.equal(mask[b], net.predict(x[b:b + 1], sets[b])[0]), b


# ------------------------------------------------------------------------------------------------
# 1. each image equals a one-image call with its own labels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,kvec", [((2, 64, 96), [1]), ((2, 64, 96), [5, 150, 7, 300]), ((3, 160, 224), [1, 2, 3]),
                                        ((3, 160, 224), [5, 150, 7, 300]), ((8, 480, 480), [5, 150, 7, 300]),
                                        ((8, 480, 480), [1, 2, 3]), ((1, 736, 736), [512])])
def test_per_image_identity(net, shape, kvec):
    B, H, W = shape
    sets = _sets([kvec[b % len(kvec)] for b in range(B)])
    x = synth.make_image(B, H, W, seed=B * 100 + H).cuda()
    _check_per_image(net, x, sets, net(x, sets), net.predict(x, sets))


def test_shared_and_repeated_labels(net):
    """Overlapping label sets (the union is encoded once) and a label repeated within one image."""
    ade = synth.ade20k_labels()
    sets = [ade[:5], ade[3:9] + ade[:2], [ade[4], ade[4], ade[0]]]
    x = synth.make_image(3, 96, 128, seed=7).cuda()
    _check_per_image(net, x, sets, net(x, sets), net.predict(x, sets))


# ------------------------------------------------------------------------------------------------
# 2. equal label sets reduce to today's call
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,K", [(3, 160, 224, 7), (8, 480, 480, 150)])
def test_uniform_sets_equal_batched_call(net, B, H, W, K):
    labels = synth.ade20k_labels()[:K]
    x = synth.make_image(B, H, W, seed=K).cuda()
    outs = net(x, [labels] * B)
    assert torch.equal(torch.cat(outs, 0), net(x, labels))
    assert torch.equal(net.predict(x, [list(labels)] * B), net.predict(x, labels))


# ------------------------------------------------------------------------------------------------
# 3. the embedding route
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,kvec", [(3, 160, 224, [5, 150, 7]), (8, 480, 480, [3, 5, 12, 20, 40, 80, 150, 150])])
def test_embedding_route(net, B, H, W, kvec):
    sets = _sets(kvec)
    x = synth.make_image(B, H, W, seed=11).cuda()
    emb = net.encode_image(x)
    for a, b in zip(net(emb, sets), net(x, sets)):
        assert torch.equal(a, b)
    assert torch.equal(net.predict(emb, sets), net.predict(x, sets))


# ------------------------------------------------------------------------------------------------
# 4. engine level: blocks at b * s equal the per-image-block path of lseg_forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 40])  # B * s = 16 (one grouped GEMM) / 320 > 256 (one GEMM per image)
def test_engine_matches_text_image_stride(net, K):
    B, H, W, s = 8, 96, 128, K
    engine = net._engine_for(torch.device("cuda"))
    feats = net._text_features(engine, synth.synthetic_prompts(B * s, seed=K))
    text = torch.zeros((engine.padded_rows(B * s) + 128, net.out_c), dtype=torch.float16, device="cuda")
    text[: B * s] = feats[: B * s]
    x = synth.make_image(B, H, W, seed=K).cuda()
    ref = engine.forward(x, text, K, text_image_stride=s)
    ref_mask = engine.forward_argmax(x, text, K, text_image_stride=s)
    logits = torch.empty((B * K, H, W), device="cuda")
    mask = torch.empty((B, H, W), dtype=torch.int64, device="cuda")
    engine.forward_ragged(x, text, [b * s for b in range(B)], [K] * B, logits=logits, mask=mask)
    assert torch.equal(logits.view(B, K, H, W), ref)
    assert torch.equal(mask, ref_mask)


# ------------------------------------------------------------------------------------------------
# 5. the GEMM stage op on integer operands: exact, and only the image's planes are written
# ------------------------------------------------------------------------------------------------
def _gemm_ragged(lib, a, text, text_row, k, out, P, sumsq=None, parts=0, scale=1.0):
    B = len(k)
    ints = C.c_int * B
    return lib.lseg_gemm_ragged(C.c_void_p(a.data_ptr()), C.c_void_p(sumsq.data_ptr()) if sumsq is not None else None,
                                parts, scale, B, P, a.shape[1], C.c_void_p(text.data_ptr()), text.shape[0],
                                ints(*text_row), ints(*k), C.c_void_p(out.data_ptr()), None)


@pytest.mark.parametrize("P,C_,k,text_row,text_rows", [
    (256, 512, [5, 150, 7, 300], [0, 234, 5, 40], 384),       # gaps, overlaps, a block that ends at the last row
    (1024, 768, [1, 129, 128], [500, 0, 1], 640),
    (128, 512, [1] * 64, list(range(64)), 64),                 # the image cap
])
def test_gemm_stage_op_exact(lib, P, C_, k, text_row, text_rows):
    from lseg_b200._lib import check
    g = torch.Generator().manual_seed(P + C_)
    B, S = len(k), 3  # S sentinel planes on each side
    a = torch.randint(-2, 3, (B * P, C_), generator=g).half().cuda()
    text = torch.randint(-2, 3, (text_rows, C_), generator=g).half().cuda()
    full = torch.full((sum(k) + 2 * S, P), float("nan"), dtype=torch.float16, device="cuda")
    check(_gemm_ragged(lib, a, text, text_row, k, full[S:], P))
    torch.cuda.synchronize()
    assert torch.isnan(full[:S]).all() and torch.isnan(full[S + sum(k):]).all()
    out, o = full[S:S + sum(k)], 0
    for b in range(B):
        ref = (text[text_row[b]:text_row[b] + k[b]].double() @ a[b * P:(b + 1) * P].double().T)
        assert torch.equal(out[o:o + k[b]].double(), ref), b
        o += k[b]


def test_gemm_stage_op_row_scale_and_cluster_modes(lib):
    """The normalised epilogue (row_sumsq / row_scale) gives the same bits in every cluster mode."""
    from lseg_b200._lib import check
    g = torch.Generator().manual_seed(5)
    k, text_row, P, C_ = [3, 200, 17], [0, 3, 100], 512, 512
    a = torch.randn((3 * P, C_), generator=g).half().cuda()
    sumsq = torch.rand((3 * P, 16), generator=g).cuda() + 0.5
    text = torch.randn((256, C_), generator=g).half().cuda()
    outs = []
    try:
        for mode in (1, 2, 3):
            check(lib.lseg_debug_set_gemm_cluster(mode))
            out = torch.full((sum(k), P), float("nan"), dtype=torch.float16, device="cuda")
            check(_gemm_ragged(lib, a, text, text_row, k, out, P, sumsq, 16, 14.3))
            outs.append(out)
    finally:
        check(lib.lseg_debug_set_gemm_cluster(2))
    assert not torch.isnan(outs[0]).any()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ------------------------------------------------------------------------------------------------
# 6. cluster modes; arch_option 1 / 2
# ------------------------------------------------------------------------------------------------
def test_cluster_modes_identical(net, lib):
    from lseg_b200._lib import check
    sets = _sets([5, 150, 7, 300])
    x = synth.make_image(4, 160, 224, seed=3).cuda()
    got = []
    try:
        for mode in (1, 2, 3):
            check(lib.lseg_debug_set_gemm_cluster(mode))
            got.append((net(x, sets), net.predict(x, sets)))
    finally:
        check(lib.lseg_debug_set_gemm_cluster(2))
    for outs, mask in got[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs, got[0][0]))
        assert torch.equal(mask, got[0][1])


@pytest.mark.parametrize("kw", [dict(arch_option=1, block_depth=2, activation="lrelu"),
                                dict(arch_option=2, block_depth=3, activation="tanh")])
def test_arch_option_per_image(kw):
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels()[:5], **{**NET_KW, **kw})
    n.load_state_dict(synth.make_state_dict(0, head_block=True))
    n = n.cuda().eval()
    sets = _sets([3, 1, 9])
    x = synth.make_image(3, 64, 96, seed=2064).cuda()
    _check_per_image(n, x, sets, n(x, sets), n.predict(x, sets))
    emb = n.encode_image(x)
    assert torch.equal(n.predict(emb, sets), n.predict(x, sets))


# ------------------------------------------------------------------------------------------------
# 7. rejections, by name, with the outputs untouched
# ------------------------------------------------------------------------------------------------
def test_rejections(net, lib):
    engine = net._engine_for(torch.device("cuda"))
    x = synth.make_image(2, 64, 96).cuda()
    emb = net.encode_image(x)
    text = torch.zeros((256, net.out_c), dtype=torch.float16, device="cuda")
    logits = torch.full((40, 64, 96), 7.0, device="cuda")
    mask = torch.full((2, 64, 96), -5, dtype=torch.int64, device="cuda")
    big = torch.full((80, 64, 1056), 7.0, device="cuda")

    def call(B=2, H=64, W=96, t=text, rows=256, text_row=(0, 10), k=(3, 4), lg=logits, mk=mask, xin=x, query=False):
        ints = C.c_int * max(1, len(k))
        tp = C.c_void_p(t.data_ptr()) if t is not None else None
        lp = C.c_void_p(lg.data_ptr()) if lg is not None else None
        mp = C.c_void_p(mk.data_ptr()) if mk is not None else None
        if query:
            rc = lib.lseg_query_ragged(engine.handle, C.c_void_p(emb.emb.data_ptr()), C.c_void_p(emb.sumsq.data_ptr()), B,
                                       H, W, tp, rows, ints(*text_row), ints(*k), lp, mp, None)
        else:
            rc = lib.lseg_forward_ragged(engine.handle, C.c_void_p(xin.data_ptr()), B, H, W, tp, rows, ints(*text_row),
                                         ints(*k), lp, mp, None)
        return rc, lib.lseg_last_error().decode()

    cases = [
        (dict(B=0, text_row=(0,), k=(1,)), "B=0"),
        (dict(B=65, text_row=(0,) * 65, k=(1,) * 65, H=64, W=96), "cap of 64"),
        (dict(k=(3, 0)), "k[1]=0"),
        (dict(text_row=(0, 253)), "text_row[1]=253 + k[1]=4 exceeds text_rows=256"),
        (dict(text_row=(-1, 0)), "text_row[0]=-1"),
        (dict(rows=40000, text_row=(0, 0), k=(40000, 40000)), "sum of k = 80000 exceeds 65535"),
        (dict(t=None), "null text"),
        (dict(lg=None, mk=None), "no output requested"),
        (dict(H=48), "multiples of 32"),
        (dict(W=1056, lg=big), "W=1056 must be <= 1024"),
    ]
    for query in (False, True):
        for kw, msg in cases:
            if query and ("H" in kw or "W" in kw or kw.get("B") == 65):
                continue  # the embedding fixes the shape
            rc, err = call(query=query, **kw)
            assert rc != 0 and msg in err, (query, kw, err)
            assert ("lseg_query_ragged" if query else "lseg_forward_ragged") in err
    torch.cuda.synchronize()
    assert (logits == 7.0).all() and (mask == -5).all() and (big == 7.0).all()
    rc = _gemm_ragged(lib, emb.emb.view(-1, net.out_c), text, [0, 0], [1, 1], text, 96)
    assert rc != 0 and "P=96" in lib.lseg_last_error().decode()


def test_python_rejections(net):
    from lseg_b200.metrics import SegmentationMetric
    x = synth.make_image(2, 64, 96).cuda()
    sets = _sets([2, 3])
    with pytest.raises(ValueError, match="out="):
        net(x, sets, out=torch.empty((2, 2, 64, 96), device="cuda"))
    with pytest.raises(ValueError, match="per-image label sets"):
        net.update_metric(SegmentationMetric(5), x, torch.zeros((2, 64, 96), dtype=torch.int64, device="cuda"), sets)
    with pytest.raises(ValueError, match="3 label sets for a batch of 2"):
        net(x, _sets([1, 1, 1]))
    with pytest.raises(ValueError, match="labelsets"):
        net.predict(x, [["a"], []])
