"""GPU tests of the recorded attention maps: the stage op lseg_attn_probs (csrc/attn_probs.cuh) against float64 with the
bound tests/probs_oracle.py derives from the kernel's rounding points, its 64-bit offsets and argument checks; the
engine's lseg_encode_image_attention (exact wiring to the hooked blocks' QKV rows, agreement with the oracle and the
reference fixture); and the drop-in's enable_attention_hooks, which must not change a single bit of anything else.

Every stage-op output lives inside an fp32 NaN-sentinel buffer that must keep its bits outside [B, heads, N, N]."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import vit_attention_oracle as A
from parity_util import NET_KW, state_dict, synth
from probs_oracle import flat_probs, probs_oracle, row_sum_bound, violations
from attention_oracle import MHSA_SHAPES
from test_attention_gpu import FAMILIES, _qkv

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
SENT = 0x7FC0DEAD  # fp32 NaN
GUARD = 4096       # sentinel elements before and after every output
STAGE_TOL = 1.0e-3  # the engine's fp32 stages against the oracle (tests/test_model_gpu.py)
HOOKED = ("attn_1", "attn_2", "attn_3", "attn_4")


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _watchdog(ops):
    yield
    torch.cuda.synchronize()
    wd = ops.read_watchdog()
    assert wd[0] == 0, f"device barrier watchdog fired: tag={wd[0]} block={wd[1]} thread={wd[2]} parity={wd[3]}"


def _guarded(shape):
    """Flat fp32 buffer: GUARD sentinels, the output, GUARD sentinels. Returns (buffer, output view)."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENT, dtype=torch.int32, device="cuda").view(torch.float32)
    return buf, buf[GUARD:GUARD + n].view(shape)


def _guards_intact(buf, n, what):
    b = buf.view(torch.int32)
    bad = int((b[:GUARD] != SENT).sum()) + int((b[GUARD + n:] != SENT).sum())
    assert bad == 0, f"{what}: {bad} sentinel elements outside the output were written"


def _check_planes(got, qkv, B, N, heads, what, flat=False):
    """Every element within the derived bound of float64, every row sum within its bound of 1."""
    x = qkv.view(B, N, 3, heads, 64)
    hc = max(1, min(heads, (1 << 24) // (N * N)))
    for b in range(B):
        for h0 in range(0, heads, hc):
            h1 = min(heads, h0 + hc)
            q, k = (x[b, :, i, h0:h1].transpose(0, 1) for i in (0, 1))  # [hc, N, 64]
            ref, bound = probs_oracle(q, k)
            g = got[b, h0:h1]
            n, msg = violations(g, ref, bound)
            assert n == 0, f"{what} image {b} heads {h0}..{h1 - 1}: {msg}"
            rs = (g.double().sum(-1) - 1).abs()
            rb = row_sum_bound(bound)
            assert bool((rs <= rb).all()), f"{what}: row sum off by {rs.max().item():.3g} > {rb.max().item():.3g}"
    if flat:
        want = flat_probs(N).item()
        assert bool((got == want).all()), f"{what}: q = 0 must give exactly fp32(1/N) = {want!r} everywhere"


# ---------------------------------------------------------------------------------------------------------------------
# 1. the stage op against float64
# ---------------------------------------------------------------------------------------------------------------------
_HEADS = [1, 2, 3, 12, 16]
EDGE = [(1 + i % 2, n, _HEADS[i % 5]) for i, n in enumerate([1, 2, 63, 64, 65, 127, 128, 129, 901, 1937, 2117])]
SHAPES = [s[:3] for s in MHSA_SHAPES if not s[3]] + EDGE


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("B,N,heads", SHAPES)
def test_probs_families(ops, B, N, heads, family):
    qkv = _qkv(family, B, N, heads, False)
    before = qkv.clone()
    shape = (B, heads, N, N)
    what = f"attn_probs B={B} N={N} heads={heads} {family}"
    buf, out = _guarded(shape)
    assert ops.attn_probs(qkv, heads, out=out) is out
    torch.cuda.synchronize()
    _guards_intact(buf, out.numel(), what)
    assert not torch.isnan(out).any(), f"{what}: NaN in the output (unwritten elements?)"
    _check_planes(out, qkv, B, N, heads, what, flat=(family == "flat"))
    again = ops.attn_probs(qkv, heads)
    assert torch.equal(again.view(torch.int32), out.view(torch.int32)), f"{what}: a second run gave other bits"
    assert torch.equal(qkv, before), f"{what}: qkv changed"
    if B > 1:
        for b in range(B):
            one = ops.attn_probs(qkv[b:b + 1].contiguous(), heads)
            assert torch.equal(one[0], out[b]), f"{what}: image {b} alone differs from its batched planes"


def test_probs_offsets_past_2_31(ops):
    """B*heads*N^2 = 480 * 2117^2 = 2.15e9 elements > 2^31 (8.6 GB): sampled rows, including the very last one, against
    float64, and the sentinels after the end untouched."""
    B, N, heads = 1, 2117, 480
    assert B * heads * N * N > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(77)
    qkv = torch.randn((B, N, 3 * heads * 64), generator=g, device="cuda").half()
    buf, out = _guarded((B, heads, N, N))
    ops.attn_probs(qkv, heads, out=out)
    torch.cuda.synchronize()
    _guards_intact(buf, out.numel(), "offsets past 2^31")
    x = qkv.view(N, 3, heads, 64)
    for h, rows in ((0, [0, N - 1]), (239, [0, 1000]), (253, [N // 2]), (heads - 1, [0, 64, N - 2, N - 1])):
        q, k = x[:, 0, h], x[:, 1, h]
        ref, bound = probs_oracle(q[rows], k)
        n, msg = violations(out[0, h, rows], ref, bound)
        assert n == 0, f"head {h} rows {rows}: {msg}"
    assert not torch.isnan(out[0, heads - 1, N - 1]).any()
    del out, buf


def _ptr(t, offset_bytes=0):
    return None if t is None else C.c_void_p(t.data_ptr() + offset_bytes)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _rejected(call, match, bufs):
    from lseg_b200._lib import LsegError, check
    before = [b.clone() for b in bufs]
    with pytest.raises(LsegError, match=match):
        check(call())
    torch.cuda.synchronize()
    for b0, b1 in zip(before, bufs):
        assert torch.equal(b0.view(torch.int32), b1.view(torch.int32)), f"rejected call ({match}) wrote its output"


def test_attn_probs_rejects(ops):
    from lseg_b200._lib import LsegError, load
    lib = load()
    B, N, heads = 2, 130, 2
    big = torch.randn((B * N * 3 * heads * 64 + 64,), device="cuda").half()
    qkv = big[:B * N * 3 * heads * 64]
    buf, out = _guarded((B, heads, N, N))

    def call(q, o, b=B, n=N, h=heads):
        return lambda: lib.lseg_attn_probs(q, o, b, n, h, _stream())

    for b, n, h, name in [(0, N, heads, "B"), (-1, N, heads, "B"), (B, 0, heads, "N"), (B, -5, heads, "N"),
                          (B, N, 0, "heads"), (B, N, -2, "heads")]:
        _rejected(call(_ptr(qkv), _ptr(out), b, n, h), f"lseg_attn_probs: {name}=-?[0-9]+ must be positive", [buf])
    # B * heads > 65535, with buffers big enough for the call, so a missing check could not fault
    Bx, hx = 4097, 16
    qx = torch.zeros((Bx * 3 * hx * 64,), dtype=torch.float16, device="cuda")
    bx, ox = _guarded((Bx, hx, 1, 1))
    _rejected(lambda: lib.lseg_attn_probs(_ptr(qx), _ptr(ox), Bx, 1, hx, _stream()), "B\\*heads = 65552", [bx])
    _rejected(call(None, _ptr(out)), "null qkv", [buf])
    _rejected(call(_ptr(qkv), None), "null out", [buf])
    _rejected(call(_ptr(big, 8), _ptr(out)), "qkv must be 16-byte aligned", [buf])
    _rejected(call(_ptr(qkv), _ptr(out, 2)), "out must be 4-byte aligned", [buf])
    # the Python wrapper checks a caller-given out, and qkv's shape
    q3 = qkv.view(B, N, 3 * heads * 64)
    for bad in (torch.zeros((B, heads, N, N), dtype=torch.float16, device="cuda"),
                torch.zeros((B, heads, N, N + 1), dtype=torch.float32, device="cuda"),
                torch.zeros((B, heads, N, 2 * N), dtype=torch.float32, device="cuda")[..., ::2]):
        before = bad.clone()
        with pytest.raises(LsegError, match="out must be a contiguous fp32"):
            ops.attn_probs(q3, heads, out=bad)
        assert torch.equal(bad, before)
    with pytest.raises(LsegError, match="qkv must be"):
        ops.attn_probs(q3, heads + 1)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the engine: lseg_encode_image_attention
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def net():
    import lseg_b200  # noqa: F401
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels(), enable_attention_hooks=True, **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


@pytest.fixture(scope="module")
def plain():
    from lseg_b200.lseg_net import LSegNet
    n = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
    n.load_state_dict(state_dict(0))
    return n.cuda().eval()


def _encode_with_hooks(eng, x, hooks):
    """lseg_encode_image_attention on a second engine over the same packed weights, created with other hook blocks."""
    from lseg_b200._lib import check, load
    lib = load()
    d = eng.weights.desc
    saved = list(d.hooks)
    for k in range(4):
        d.hooks[k] = hooks[k]
    h = C.c_void_p()
    try:
        check(lib.lseg_create(C.byref(d), torch.cuda.current_device(), C.byref(h)))
    finally:
        for k in range(4):
            d.hooks[k] = saved[k]
    try:
        B, _, H, W = x.shape
        shape = eng.attention_shape(B, H, W)
        attn = [torch.empty(shape, dtype=torch.float32, device="cuda") for _ in range(4)]
        emb = torch.empty((B, H // 2, W // 2, eng.out_c), dtype=torch.float16, device="cuda")
        sumsq = torch.empty((B, H // 2, W // 2, eng.out_c // 32), dtype=torch.float32, device="cuda")
        ptrs = (C.c_void_p * 4)(*[a.data_ptr() for a in attn])
        check(lib.lseg_encode_image_attention(h, _ptr(x), B, H, W, _ptr(emb), _ptr(sumsq), ptrs, _stream()))
        torch.cuda.synchronize()
    finally:
        lib.lseg_destroy(h)
    return attn


def test_engine_wiring_exact(ops, net):
    """With hooks (0, 1, 2, 3), attn_1 is lseg_attn_probs on block 0's QKV rows rebuilt from stage ops (patchify -> patch
    GEMM -> assemble_tokens -> LayerNorm -> QKV GEMM), bit for bit: the step reads the right block's rows."""
    sd = state_dict(0)
    eng = net._engine_for(torch.device("cuda"))
    B, H, W = 2, 64, 96
    x = synth.make_image(B, H, W, seed=2064).cuda()
    attn = _encode_with_hooks(eng, x, (0, 1, 2, 3))
    p = "pretrained.model."
    D, gh, gw = 1024, H // 16, W // 16
    T, N = gh * gw, gh * gw + 1
    a = ops.patchify(x)
    pw = ops.pad_rows(sd[p + "patch_embed.proj.weight"].reshape(D, -1).cuda().half())
    patch = torch.empty((B * T, D), dtype=torch.float32, device="cuda")
    ops.gemm(a, pw, D, bias=sd[p + "patch_embed.proj.bias"].float().cuda(), out_f32=patch)
    pos = ops.pos_resize(sd[p + "pos_embed"].reshape(-1, D).float().cuda().contiguous(), 24, gh, gw)
    xt = ops.assemble_tokens(patch, sd[p + "cls_token"].reshape(D).float().cuda().contiguous(), pos, B, T)
    b0 = p + "blocks.0."
    xn = ops.layernorm(xt.view(B * N, D), sd[b0 + "norm1.weight"].float().cuda(), sd[b0 + "norm1.bias"].float().cuda(),
                       1e-6)
    qkv = torch.empty((B * N, 3 * D), dtype=torch.float16, device="cuda")
    ops.gemm(xn, sd[b0 + "attn.qkv.weight"].cuda().half().contiguous(), 3 * D,
             bias=sd[b0 + "attn.qkv.bias"].float().cuda(), out_f16=qkv, ldc=3 * D)
    want = ops.attn_probs(qkv.view(B, N, 3 * D), 16)
    torch.cuda.synchronize()
    assert torch.equal(attn[0].view(torch.int32), want.view(torch.int32))
    # the other hooked blocks are different blocks: different maps
    for k in range(1, 4):
        assert not torch.equal(attn[k], attn[0])


def _engine_bound(q, k, rows, w_ref):
    """|engine - oracle| bound on rows `rows` of the attention [B, heads, N, N] from named error sources:
      (1) the engine stores q and k in fp16: 2^-11 relative per element;
      (2) the trunk that produced them: the engine's fp32 stages agree with the oracle's to STAGE_TOL of the stage's
          largest magnitude (tests/test_model_gpu.py), charged here to q and k relative to their plane's largest entry;
      (3) the kernel's own rounding points: the bound of tests/probs_oracle.py on the fp16 q, k.
    With e = 2^-11 + STAGE_TOL, a score 0.125 q.k moves by at most
      delta_i = 0.125 (2^-10 sum_d |q_d k_d| + e (Qmax ||k_j||_1 + Kmax ||q_i||_1) + e^2 64 Qmax Kmax),
    and a softmax row whose scores move by at most delta moves each probability by at most w (exp(2 delta) - 1)."""
    qd, kd = q.double(), k.double()
    qr = qd[:, :, rows]
    qmax = qd.abs().amax(dim=(-2, -1), keepdim=True)  # [B, heads, 1, 1]
    kmax = kd.abs().amax(dim=(-2, -1), keepdim=True)
    e = 2.0 ** -11 + STAGE_TOL
    A_ = (qr.abs() @ kd.abs().transpose(-1, -2)).amax(-1, keepdim=True)  # [B, heads, rows, 1]
    k1 = kd.abs().sum(-1).amax(-1, keepdim=True).unsqueeze(-1)            # [B, heads, 1, 1]
    q1 = qr.abs().sum(-1, keepdim=True)                                   # [B, heads, rows, 1]
    delta = 0.125 * (2.0 ** -10 * A_ + e * (qmax * k1 + kmax * q1) + e * e * 64 * qmax * kmax)
    _, kernel = probs_oracle(qr.half(), k.half())
    return w_ref * torch.expm1(2 * delta) + kernel


@pytest.mark.parametrize("tag,B,H,W,seed", [("small", 2, 64, 96, 2064), ("s480", 1, 480, 480, 1480)])
def test_engine_against_oracle_and_reference(net, tag, B, H, W, seed):
    z = np.load(os.path.join(GOLD, "ref_attention.npz"))
    x = synth.make_image(B, H, W, seed=seed)
    qk = {}
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
    ora = A.vit_attention_maps(x, state_dict(0), qk_out=qk)
    net.encode_image(x.cuda())
    N = (H // 16) * (W // 16) + 1
    rows = list(range(N)) if tag == "small" else [int(r) for r in z["s480_rows"]]
    worst = 0.0
    for name in HOOKED:
        got = net.pretrained.attention[name]
        assert got.shape == (B, 16, N, N) and got.dtype == torch.float32 and got.is_cuda
        got = got[:, :, rows].cpu().double()
        q, k = qk[name]
        w_ref = ora[name][:, :, rows].double()
        bound = _engine_bound(q, k, rows, w_ref)
        for ref in (w_ref, torch.from_numpy(z[f"{tag}_{name}"]).double()):
            err = (got - ref).abs()
            assert bool((err <= bound).all()), f"{tag} {name}: worst |err| / bound {(err / bound).max().item():.3f}"
            worst = max(worst, (err / bound).max().item())
    print(f"{tag}: worst |engine - oracle| / bound = {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. the drop-in: nothing else changes
# ---------------------------------------------------------------------------------------------------------------------
def _labels(k):
    return synth.tokenize(synth.ade20k_labels()[:k])


@pytest.mark.parametrize("K", [2, 150])
def test_flag_changes_no_output(net, plain, K):
    from lseg_b200.metrics import SegmentationMetric
    x = synth.make_image(2, 160, 224, seed=K).cuda()
    tokens = _labels(K)
    net.pretrained.attention.clear()
    assert torch.equal(net(x, tokens), plain(x, tokens))
    assert sorted(net.pretrained.attention) == list(HOOKED)
    assert torch.equal(net.predict(x, tokens), plain.predict(x, tokens))
    target = torch.randint(-1, K, (2, 160, 224), generator=torch.Generator().manual_seed(3)).cuda()
    m_a, m_b = SegmentationMetric(K), SegmentationMetric(K)
    net.update_metric(m_a, x, target, tokens)
    plain.update_metric(m_b, x, target, tokens)
    assert torch.equal(m_a.stats, m_b.stats) and int(m_a.stats.sum()) > 0
    e_a, e_b = net.encode_image(x), plain.encode_image(x)
    assert torch.equal(e_a.emb, e_b.emb) and torch.equal(e_a.sumsq, e_b.sumsq)
    out = torch.full((2, K, 160, 224), float("nan"), device="cuda")
    assert net(x, tokens, out=out) is out and torch.equal(out, plain(x, tokens))
    # per-image label sets
    sets = [synth.ade20k_labels()[:3], synth.ade20k_labels()[5:12]]
    for a, b in zip(net(x, sets), plain(x, sets)):
        assert torch.equal(a, b)
    assert torch.equal(net.predict(x, sets), plain.predict(x, sets))


def test_flag_launches(net, plain):
    """A forward without the flag runs the launches it ran before; the recording encode runs four more than encode."""
    x = synth.make_image(1, 64, 96, seed=1).cuda()
    tokens = _labels(3)
    pe = plain._engine_for(torch.device("cuda"))
    plain(x, tokens)
    n_forward = pe.last_launch_count()
    plain.encode_image(x)
    n_encode = pe.last_launch_count()
    emb, sumsq, attn = pe.encode_image_attention(x)  # the recording plan lives beside the plain one on this engine
    assert pe.last_launch_count() == n_encode + 4
    plain(x, tokens)
    assert pe.last_launch_count() == n_forward
    e2, s2 = pe.encode_image(x)
    assert pe.last_launch_count() == n_encode
    assert torch.equal(emb, e2) and torch.equal(sumsq, s2)


def test_per_image_independence(net):
    x = synth.make_image(3, 96, 128, seed=33).cuda()
    net.encode_image(x)
    batched = dict(net.pretrained.attention)
    for b in range(3):
        net.encode_image(x[b:b + 1])
        for name in HOOKED:
            assert torch.equal(net.pretrained.attention[name][0], batched[name][b]), (b, name)


def test_fresh_tensors_and_embedding_queries(net):
    """Every image-path call stores new tensors (ones a caller kept are never overwritten); a query on a PixelEmbedding
    runs no trunk and leaves the dict as it is."""
    x1 = synth.make_image(1, 64, 96, seed=4).cuda()
    x2 = synth.make_image(1, 64, 96, seed=5).cuda()
    emb = net.encode_image(x1)
    kept = net.pretrained.attention
    first = {k: v for k, v in kept.items()}
    copies = {k: v.clone() for k, v in first.items()}
    net.predict(x2, _labels(3))
    assert net.pretrained.attention is kept  # the same dict, new entries
    for name in HOOKED:
        assert kept[name] is not first[name]
        assert torch.equal(first[name], copies[name])
        assert not torch.equal(kept[name], first[name])
    now = {k: v for k, v in kept.items()}
    net(emb, _labels(3))
    net.predict(emb, _labels(3))
    assert all(kept[k] is now[k] for k in HOOKED) and sorted(kept) == list(HOOKED)


def test_zero_shot_and_rn50x16():
    from lseg_b200.lseg_net import LSegNet, LSegNetZS
    from lseg_b200.metrics import FewShotMeter
    names = [f"class {i}" for i in range(20)]
    nets = []
    for flag in (True, False):
        n = LSegNetZS(label_list=names, enable_attention_hooks=flag, **NET_KW)
        n.load_state_dict(state_dict(0))
        nets.append(n.cuda().eval())
    x = synth.make_image(4, 96, 128, seed=5).cuda()
    ci = torch.tensor([3, 7, 3, 19])
    assert torch.equal(nets[0](x, ci), nets[1](x, ci))
    assert sorted(nets[0].pretrained.attention) == list(HOOKED)
    assert torch.equal(nets[0].predict(x, ci), nets[1].predict(x, ci))
    target = torch.randint(-1, 2, (4, 96, 128), generator=torch.Generator().manual_seed(2)).cuda()
    m = [FewShotMeter(20, [3, 7, 19]) for _ in range(2)]
    for n, mm in zip(nets, m):
        n.update_metric(mm, x, ci.cuda(), target)
    assert torch.equal(m[0].stats, m[1].stats) and int(m[0].stats.sum()) > 0
    bb = "clipRN50x16_vitl16_384"
    pair = []
    for flag in (True, False):
        n = LSegNet(labels=synth.ade20k_labels(), enable_attention_hooks=flag, **{**NET_KW, "backbone": bb})
        n.load_state_dict(state_dict(0, bb))
        pair.append(n.cuda().eval())
    tokens = _labels(7)
    x = synth.make_image(2, 160, 224, seed=7).cuda()
    assert torch.equal(pair[0](x, tokens), pair[1](x, tokens))
    assert torch.equal(pair[0].predict(x, tokens), pair[1].predict(x, tokens))
    a = pair[0].pretrained.attention["attn_1"]
    assert a.shape == (2, 16, 141, 141)
    assert (a.double().sum(-1) - 1).abs().max().item() < 1e-4


def test_flag_is_a_noop_on_b32_and_rn101():
    from lseg_b200.lseg_net import LSegNet, LSegRNNetZS
    bb = "clip_vitb32_384"
    pair = []
    for flag in (True, False):
        n = LSegNet(labels=synth.ade20k_labels(), enable_attention_hooks=flag, **{**NET_KW, "backbone": bb})
        n.load_state_dict(state_dict(0, bb))
        pair.append(n.cuda().eval())
    x = synth.make_image(2, 160, 224, seed=8).cuda()
    tokens = _labels(5)
    assert torch.equal(pair[0](x, tokens), pair[1](x, tokens))
    assert not hasattr(pair[0].pretrained, "attention")
    names = [f"class {i}" for i in range(20)]
    rn = []
    for flag in (True, False):
        n = LSegRNNetZS(label_list=names, features=256, arch_option=0, block_depth=0, activation="lrelu",
                        enable_attention_hooks=flag)
        n.load_state_dict(state_dict(0, "clip_resnet101"))
        rn.append(n.cuda().eval())
    x = synth.make_image(2, 96, 128, seed=9).cuda()
    ci = torch.tensor([1, 2])
    assert torch.equal(rn[0](x, ci), rn[1](x, ci))
    assert not hasattr(rn[0].pretrained, "attention")
    # the engine refuses to record on the ResNet trunk, by name, before anything runs
    from lseg_b200._lib import LsegError
    eng = rn[0]._engine_for(torch.device("cuda"))
    with pytest.raises(ValueError, match="ViT trunk"):
        eng.encode_image_attention(x)
    from lseg_b200._lib import load
    lib = load()
    bufs = [torch.full((16,), SENT, dtype=torch.int32, device="cuda").view(torch.float32) for _ in range(4)]
    emb = torch.empty((2, 48, 64, 512), dtype=torch.float16, device="cuda")
    sq = torch.empty((2, 48, 64, 16), dtype=torch.float32, device="cuda")
    ptrs = (C.c_void_p * 4)(*[b.data_ptr() for b in bufs])
    from lseg_b200._lib import check
    with pytest.raises(LsegError, match="no ViT trunk"):
        check(lib.lseg_encode_image_attention(eng.handle, _ptr(x), 2, 96, 128, _ptr(emb), _ptr(sq), ptrs, _stream()))
    for b in bufs:
        assert bool((b.view(torch.int32) == SENT).all())


def test_encode_image_attention_rejects(net):
    from lseg_b200._lib import LsegError, check, load
    lib = load()
    eng = net._engine_for(torch.device("cuda"))
    B, H, W = 1, 64, 96
    x = synth.make_image(B, H, W, seed=1).cuda()
    shape = eng.attention_shape(B, H, W)
    bufs = [_guarded(shape) for _ in range(4)]
    emb = torch.full((B, H // 2, W // 2, 512), 7.0, dtype=torch.float16, device="cuda")
    sq = torch.full((B, H // 2, W // 2, 16), 7.0, dtype=torch.float32, device="cuda")
    watch = [b for b, _ in bufs] + [emb, sq]

    def call(ptrs, xp=_ptr(x), b=B, h=H, w=W):
        arr = (C.c_void_p * 4)(*ptrs)
        return lambda: lib.lseg_encode_image_attention(eng.handle, xp, b, h, w, _ptr(emb), _ptr(sq), arr, _stream())

    good = [o.data_ptr() for _, o in bufs]
    for k in range(4):
        p = list(good)
        p[k] = None
        _rejected_any(call(p), f"null attn\\[{k}\\]", watch)
        p[k] = good[k] + 2
        _rejected_any(call(p), f"attn\\[{k}\\] must be 4-byte aligned", watch)
    _rejected_any(lambda: lib.lseg_encode_image_attention(eng.handle, _ptr(x), B, H, W, _ptr(emb), _ptr(sq), None,
                                                          _stream()), "null attn", watch)
    _rejected_any(call(good, b=0), "B=0", watch)
    _rejected_any(call(good, h=70), "multiples of 32", watch)
    _rejected_any(call(good, xp=None), "null x", watch)
    with pytest.raises(LsegError):
        check(lib.lseg_encode_image_attention(None, _ptr(x), B, H, W, _ptr(emb), _ptr(sq),
                                              (C.c_void_p * 4)(*good), _stream()))


def _rejected_any(call, match, bufs):
    from lseg_b200._lib import LsegError, check
    before = [b.clone() for b in bufs]
    with pytest.raises(LsegError, match=match):
        check(call())
    torch.cuda.synchronize()
    for b0, b1 in zip(before, bufs):
        assert torch.equal(b0.view(torch.uint8), b1.view(torch.uint8)), f"rejected call ({match}) wrote an output"
