"""GPU parity tests of the stage ops (C ABI) against plain torch fp32 references of the same op.

Tolerances: operands are fp16 (inputs are pre-rounded so the reference sees identical values),
accumulation is fp32 on both sides -> differences come only from summation order (<= 1e-3 relative
to the output scale) plus one fp16 rounding where the output is fp16 (2^-11 relative).
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


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


def _rand(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _close(got, ref, tol, what):
    got = got.float()
    ref = ref.float()
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    denom = ref.abs().max().item() + 1e-12
    err = (got - ref).abs().max().item() / denom
    assert err <= tol, f"{what}: max rel err {err:.3e} > {tol:.1e} (scale {denom:.3e})"


@pytest.mark.parametrize("M,N,K", [(300, 256, 128), (7208, 3072, 1024), (500, 128, 512), (1000, 512, 4096),
                                   (8, 1024, 1024), (154, 1536, 512)])
def test_gemm_bias_f32_f16(ops, M, N, K):
    a = _rand((M, K), 1)
    w = _rand((N, K), 2, 0.05)
    bias = _rand((N,), 3, 1.0, torch.float32)
    ref = a.float() @ w.float().t() + bias
    out32 = torch.zeros((M, N), dtype=torch.float32, device="cuda")
    out16 = torch.zeros((M, N), dtype=torch.float16, device="cuda")
    a_pad = ops.pad_rows(a)  # rows >= 128 so the TMA box never exceeds the tensor
    ops.gemm(a_pad, ops.pad_rows(w), N, M=M, bias=bias, out_f32=out32, out_f16=out16)
    _close(out32, ref, 2e-4, "fp32 out")
    _close(out16, ref, 1e-3, "fp16 out")


@pytest.mark.parametrize("M,N,K", [(7208, 1024, 1024), (7208, 1024, 4096), (8468, 1024, 1024), (300, 1024, 512)])
def test_gemm_inplace_residual_tile_widths(ops, M, N, K):
    """x += A W^T + b through the bulk reduce-add epilogue at the ViT shapes: B=8 480^2 (29 row pairs -> the planner picks
    224-wide tiles: 145 pair tiles = 1.96 waves), B=4 736^2 (34 row pairs -> 256-wide), and a single-wave case. The column
    split of the 224-wide tile (128 | 96 per epilogue warp pair, last tile 128 valid columns) must cover every column."""
    a = _rand((M, K), 41, 0.5)
    w = _rand((N, K), 42, 0.03)
    bias = _rand((N,), 43, 0.5, torch.float32)
    res = _rand((M, N), 44, 1.0, torch.float32)
    x = res.clone()
    ops.gemm(ops.pad_rows(a), ops.pad_rows(w), N, M=M, bias=bias, res_f32=x, out_f32=x)
    _close(x, a.float() @ w.float().t() + bias + res, 2e-4, f"in-place residual {M}x{N}x{K}")


def test_gemm_gelu_residual_relu(ops):
    M, N, K = 901 * 2, 1024, 1024
    a = _rand((M, K), 4)
    w = _rand((N, K), 5, 0.03)
    bias = _rand((N,), 6, 0.5, torch.float32)
    res = _rand((M, N), 7, 1.0, torch.float32)
    res2 = _rand((M, N), 8, 1.0, torch.float32)
    scale = _rand((N,), 9, 1.0, torch.float32).abs() + 0.5
    wp = ops.pad_rows(w)
    # GELU(erf) epilogue, fp16 out
    out16 = torch.zeros((M, N), dtype=torch.float16, device="cuda")
    ops.gemm(a, wp, N, bias=bias, act=ops.ACT_GELU, out_f16=out16)
    _close(out16, F.gelu(a.float() @ w.float().t() + bias), 1e-3, "gelu")
    # scale + bias + two fp32 residuals, in-place on res, plus relu copy
    acc = (a.float() @ w.float().t()) * scale + bias + res + res2
    x = res.clone()
    relu16 = torch.zeros((M, N), dtype=torch.float16, device="cuda")
    ops.gemm(a, wp, N, bias=bias, scale=scale, res_f32=x, res2_f32=res2, out_f32=x, out_f16_relu=relu16)
    _close(x, acc, 2e-4, "scale/bias/res in-place")
    _close(relu16, acc.clamp_min(0), 1e-3, "relu copy")
    # in-place fp32 residual stream x += A W^T + b (bulk tensor reduce-add epilogue), M not a tile multiple
    x2 = res.clone()
    ops.gemm(a, wp, N, bias=bias, res_f32=x2, out_f32=x2)
    _close(x2, a.float() @ w.float().t() + bias + res, 2e-4, "in-place residual (reduce-add)")
    # grouped (per-image) bias rows
    gb = _rand((2, N), 10, 1.0, torch.float32)
    out32 = torch.zeros((M, N), dtype=torch.float32, device="cuda")
    ops.gemm(a, wp, N, bias=gb, bias_group_rows=901, out_f32=out32)
    ref = a.float() @ w.float().t() + gb.repeat_interleave(901, dim=0)
    _close(out32, ref, 2e-4, "grouped bias")
    # QuickGELU + fp16 residual stream (CLIP text tower semantics)
    r16 = _rand((M, N), 11)
    out16 = torch.zeros((M, N), dtype=torch.float16, device="cuda")
    ops.gemm(a, wp, N, bias=bias, res_f16=r16, out_f16=out16)
    ref = (r16 + (a.float() @ w.float().t() + bias).half()).float()
    _close(out16, ref, 1.5e-3, "fp16 residual")
    ops.gemm(a, wp, N, bias=bias, act=ops.ACT_QUICKGELU, out_f16=out16)
    h = (a.float() @ w.float().t() + bias).half()
    _close(out16, (h * torch.sigmoid(1.702 * h)).float(), 2e-3, "quickgelu")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 30, 30, 128, 256), (1, 15, 15, 1024, 256), (2, 120, 120, 256, 256),
                                            (3, 60, 60, 512, 256)])
def test_conv3x3(ops, B, H, W, Cin, Cout):
    x = _rand((B, H, W, Cin), 12)
    wt = _rand((Cout, Cin, 3, 3), 13, 0.03)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), padding=1).permute(0, 2, 3, 1)
    wp = ops.pad_rows(wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous())  # tap-major [N, (ky,kx,c)]
    out32 = torch.zeros((B, H, W, Cout), dtype=torch.float32, device="cuda")
    relu16 = torch.zeros((B, H, W, Cout), dtype=torch.float16, device="cuda")
    ops.gemm(x, wp, Cout, conv=(3, 1), out_f32=out32, out_f16_relu=relu16, ldc=Cout)
    _close(out32, ref, 3e-4, "conv3x3")
    _close(relu16, ref.clamp_min(0), 1e-3, "conv3x3 relu copy")


@pytest.mark.parametrize("B,H,W,Cin", [(8, 15, 15, 256), (8, 30, 30, 256), (8, 15, 15, 1024), (1, 30, 30, 1024)])
def test_conv3x3_split_k_epilogues(ops, B, H, W, Cin):
    """Low-resolution decoder convs run as deterministic split-K (raw fp32 partials + splitk_reduce_kernel): the reduce
    applies the whole RCU epilogue — folded-BN scale / shift, ReLU, two fp32 residuals, fp32 + fp16 + relu-fp16 outputs —
    and two runs give the same bits."""
    Cout = 256
    x = _rand((B, H, W, Cin), 52)
    wt = _rand((Cout, Cin, 3, 3), 53, 0.03)
    scale = _rand((Cout,), 54, 0.2, torch.float32) + 1.0
    shift = _rand((Cout,), 55, 0.3, torch.float32)
    r1 = _rand((B, H, W, Cout), 56, 1.0, torch.float32)
    r2 = _rand((B, H, W, Cout), 57, 1.0, torch.float32)
    conv = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), padding=1).permute(0, 2, 3, 1)
    wp = ops.pad_rows(wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous())
    # conv1 of an RCU: relu(bn(conv)) -> fp16
    t16 = torch.zeros((B, H, W, Cout), dtype=torch.float16, device="cuda")
    ops.gemm(x, wp, Cout, conv=(3, 1), scale=scale, bias=shift, act=ops.ACT_RELU, out_f16=t16, ldc=Cout)
    _close(t16, (conv * scale + shift).clamp_min(0), 1e-3, "split-K conv + bn + relu")
    # conv2 of an RCU: bn(conv) + x + skip -> fp32, fp16, relu-fp16
    o32 = torch.zeros((B, H, W, Cout), dtype=torch.float32, device="cuda")
    o16 = torch.zeros((B, H, W, Cout), dtype=torch.float16, device="cuda")
    orl = torch.zeros((B, H, W, Cout), dtype=torch.float16, device="cuda")
    ops.gemm(x, wp, Cout, conv=(3, 1), scale=scale, bias=shift, res_f32=r1, res2_f32=r2, out_f32=o32, out_f16=o16,
             out_f16_relu=orl, ldc=Cout)
    ref = conv * scale + shift + r1 + r2
    _close(o32, ref, 3e-4, "split-K conv + residuals fp32")
    _close(o16, ref, 1e-3, "split-K conv + residuals fp16")
    _close(orl, ref.clamp_min(0), 1e-3, "split-K conv + residuals relu fp16")
    again = torch.zeros_like(o32)
    ops.gemm(x, wp, Cout, conv=(3, 1), scale=scale, bias=shift, res_f32=r1, res2_f32=r2, out_f32=again, ldc=Cout)
    assert torch.equal(again, o32), "split-K reduction is not deterministic"


def test_resnet_glue_and_bottleneck_epilogue(ops):
    """The ResNet-101 trunk's pieces against torch: stem rows (7x7 s2 p3 im2col + GEMM + folded BN + ReLU), max pool,
    1x1 stride-2 subsampling, 3x3 stride-2 conv, and the bottleneck's closing GEMM relu(bn3(conv3) + identity) with the
    fp32 stream updated in place."""
    B, H, W = 2, 64, 96
    x = _rand((B, 3, H, W), 71, 1.0, torch.float32)
    wt = _rand((64, 3, 7, 7), 72, 0.05)
    scale = _rand((64,), 73, 0.2, torch.float32) + 1.0
    shift = _rand((64,), 74, 0.3, torch.float32)
    a = ops.stem_im2col(x)
    assert a.shape == (B * (H // 2) * (W // 2), 192) and float(a[:, 147:].abs().max()) == 0.0
    wp = torch.zeros((128, 192), dtype=torch.float16, device="cuda")
    wp[:64, :147] = wt.reshape(64, 147)
    stem = torch.zeros((a.shape[0], 64), dtype=torch.float16, device="cuda")
    ops.gemm(a, wp, 64, scale=scale, bias=shift, act=ops.ACT_RELU, out_f16=stem)
    ref = F.relu(F.conv2d(x.half().float(), wt.float(), stride=2, padding=3) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    _close(stem.view(B, H // 2, W // 2, 64), ref.permute(0, 2, 3, 1), 1e-3, "stem conv")
    # stage-1 shapes: K = 64 (a single 64-wide K chunk) and N = 64 (half of the narrowest tile)
    w1 = _rand((64, 64), 82, 0.1)
    o1 = torch.zeros((stem.shape[0], 64), dtype=torch.float16, device="cuda")
    ops.gemm(stem, ops.pad_rows(w1), 64, scale=scale, bias=shift, act=ops.ACT_RELU, out_f16=o1)
    _close(o1, F.relu((stem.float() @ w1.float().t()) * scale + shift), 1e-3, "1x1 conv K=64 N=64")
    c64 = torch.zeros((B, H // 2, W // 2, 64), dtype=torch.float16, device="cuda")
    w64 = _rand((64, 64, 3, 3), 83, 0.05)
    ops.gemm(stem.view(B, H // 2, W // 2, 64), ops.pad_rows(w64.permute(0, 2, 3, 1).reshape(64, 9 * 64).contiguous()), 64,
             conv=(3, 1), out_f16=c64, ldc=64)
    _close(c64, F.conv2d(stem.view(B, H // 2, W // 2, 64).float().permute(0, 3, 1, 2), w64.float(), padding=1).permute(0, 2, 3, 1),
           1e-3, "3x3 conv C=64 N=64")
    pooled = ops.maxpool3x3s2_nhwc(stem.view(B, H // 2, W // 2, 64))
    want = F.max_pool2d(stem.view(B, H // 2, W // 2, 64).float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(pooled.float(), want)
    t = _rand((B, 16, 24, 128), 75)
    assert torch.equal(ops.subsample2_nhwc(t), t[:, ::2, ::2].contiguous())
    # 3x3 stride-2 conv = im2col rows + GEMM
    w2 = _rand((128, 128, 3, 3), 76, 0.03)
    rows = ops.im2col_3x3_s2(t)
    o2 = torch.zeros((rows.shape[0], 128), dtype=torch.float16, device="cuda")
    ops.gemm(rows, ops.pad_rows(w2.permute(0, 2, 3, 1).reshape(128, 9 * 128).contiguous()), 128, out_f16=o2)
    _close(o2.view(B, 8, 12, 128), F.conv2d(t.float().permute(0, 3, 1, 2), w2.float(), stride=2, padding=1).permute(0, 2, 3, 1),
           1e-3, "3x3 stride-2 conv")
    # closing GEMM of a bottleneck: in-place fp32 stream + fp16 copy, ReLU after the residual add
    M, K, N = B * 8 * 12 * 4, 128, 512
    t2 = _rand((M, K), 77)
    w3 = _rand((N, K), 78, 0.05)
    s3 = _rand((N,), 79, 0.2, torch.float32) + 1.0
    b3 = _rand((N,), 80, 0.3, torch.float32)
    stream = _rand((M, N), 81, 1.0, torch.float32)
    want = F.relu((t2.float() @ w3.float().t()) * s3 + b3 + stream)
    y16 = torch.zeros((M, N), dtype=torch.float16, device="cuda")
    ops.gemm(t2, ops.pad_rows(w3), N, scale=s3, bias=b3, res_f32=stream, out_f32=stream, out_f16=y16, relu_after_res=True)
    _close(stream, want, 3e-4, "bottleneck output fp32 (in place)")
    _close(y16, want, 1e-3, "bottleneck output fp16")
    assert float(stream.min()) >= 0.0


@pytest.mark.parametrize("s,cin,cout,g", [(4, 256, 256, 30), (2, 512, 512, 6)])
def test_deconv_depth_to_space(ops, s, cin, cout, g):
    B = 2
    x = _rand((B * g * g, cin), 14)
    wt = _rand((cin, cout, s, s), 15, 0.05)  # ConvTranspose2d weight layout [Cin, Cout, kH, kW]
    bias = _rand((cout,), 16, 1.0, torch.float32)
    xin = x.float().view(B, g, g, cin).permute(0, 3, 1, 2)
    ref = F.conv_transpose2d(xin, wt.float(), bias, stride=s).permute(0, 2, 3, 1)  # NHWC
    wp = ops.pad_rows(wt.permute(2, 3, 1, 0).reshape(s * s * cout, cin).contiguous())  # [(i,j,co), ci]
    bexp = bias.repeat(s * s).contiguous()
    out = torch.zeros((B, g * s, g * s, cout), dtype=torch.float16, device="cuda")
    ops.gemm(x, wp, s * s * cout, bias=bexp, out_f16=out, store=ops.STORE_D2S, d2s=(s, cout, g, g))
    _close(out, ref, 1e-3, "deconv d2s")


@pytest.mark.parametrize("K", [2, 150, 512])
def test_gemm_nchw_store(ops, K):
    B, P = 2, 57600 // 16
    a = _rand((B * P, 512), 17)
    t = _rand((K, 512), 18, 0.05)
    out = torch.zeros((B, K, P), dtype=torch.float16, device="cuda")
    ops.gemm(a, ops.pad_rows(t), K, out_f16=out, store=ops.STORE_NCHW_T, nchw=(P, K))
    ref = (a.float() @ t.float().t()).view(B, P, K).permute(0, 2, 1)
    _close(out, ref, 1e-3, "nchw store")


def test_deferred_row_normalisation(ops):
    """head1 -> pixel x text with the L2 normalisation deferred into the second GEMM's epilogue
    (lseg_net.py:185-196): logits = logit_scale * (x / ||x||) . t"""
    B, P, K = 2, 1280, 150
    path = _rand((B * P, 256), 40)
    w1 = _rand((512, 256), 41, 0.06)
    b1 = _rand((512,), 42, 0.05, torch.float32)
    t = _rand((K, 512), 43, 0.05)
    t = (t.float() / t.float().norm(dim=-1, keepdim=True)).half()
    feat16 = torch.zeros((B * P, 512), dtype=torch.float16, device="cuda")
    sumsq = torch.zeros((B * P, 16), dtype=torch.float32, device="cuda")  # [row, 512/32] partial sums
    ops.gemm(path, ops.pad_rows(w1), 512, bias=b1, out_f16=feat16, out_row_sumsq=sumsq)
    x = path.float() @ w1.float().t() + b1
    _close(sumsq, (x * x).view(B * P, 16, 32).sum(-1), 1e-4, "row sumsq parts")
    out = torch.zeros((B, K, P), dtype=torch.float16, device="cuda")
    ls = math.exp(math.log(1 / 0.07))
    ops.gemm(feat16, ops.pad_rows(t), K, out_f16=out, store=ops.STORE_NCHW_T, nchw=(P, K), row_sumsq=sumsq,
             row_scale=ls)
    img = (x / x.norm(dim=-1, keepdim=True)).half()
    ref = ((torch.tensor(ls) * img) @ t.t()).float().view(B, P, K).permute(0, 2, 1)  # the reference's fp16 recipe
    _close(out, ref, 2e-3, "deferred normalisation vs reference recipe")


def _mhsa_ref(qkv, B, N, heads, causal):
    D = heads * 64
    q, k, v = qkv.float().view(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * 0.125
    if causal:
        s = s + torch.full((N, N), float("-inf"), device="cuda").triu_(1)
    return (s.softmax(-1) @ v).transpose(1, 2).reshape(B * N, D)


MHSA_SHAPES = [
    (2, 901, 16, False, 1.0), (3, 77, 8, True, 1.0), (1, 37, 16, False, 1.0), (1, 300, 2, True, 1.0),
    # tile-boundary cases of the 64-key two-stream kernels: one tile only (second stream empty), exact multiples,
    # 1..2 keys in the tail tile, odd/even tile counts; amp 3 makes the running-max offset move (O rescale path)
    (1, 64, 1, False, 1.0), (1, 65, 1, True, 1.0), (1, 128, 2, False, 1.0), (1, 130, 2, False, 3.0),
    (1, 1025, 2, False, 1.0), (2, 300, 2, False, 3.0), (1, 193, 1, True, 3.0),
    # token counts of BASELINE.json configs[4]: 704^2 -> 1937, 736^2 -> 2117 (34 key tiles; 17 query tiles)
    (1, 1937, 4, False, 1.0), (1, 2117, 3, False, 1.0), (1, 2117, 1, False, 3.0)]


# variant None = the kernel the engine runs; 0..8 = every number lseg_mhsa_variant accepts: 0/1/2/5/6 all exponentials
# on the MUFU pipe, 3/7 one of four score pairs on the FMA pipe, 4/8 two of four (include/lseg_b200.h)
@pytest.mark.parametrize("variant", [None, 0, 1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("B,N,heads,causal,amp", MHSA_SHAPES)
def test_mhsa(ops, B, N, heads, causal, amp, variant):
    D = heads * 64
    qkv = _rand((B, N, 3 * D), 19, amp)
    out = ops.mhsa(qkv, B, N, heads, causal, variant=variant)
    _close(out, _mhsa_ref(qkv, B, N, heads, causal), 2e-3, f"mhsa variant {variant}")


def test_text_attn_rounding_points(ops):
    """lseg_text_attn follows torch's multi_head_attention_forward on fp16 tensors step by step (q scaled in fp16, bmm ->
    fp16, softmax -> fp16 normalised, bmm -> fp16): against that recipe evaluated with the same rounding points the result
    is bit-identical except where an fp32 sum formed in another order lands on the other side of an fp16 rounding
    boundary (rare 1-ulp differences)."""
    K, L, heads = 23, 77, 8
    D = heads * 64
    qkv = _rand((K, L, 3 * D), 31, 1.5)
    got = ops.text_attn(qkv, K, L, heads).float()

    def r16(t):
        return t.half().float()
    q, k, v = qkv.float().view(K, L, 3, heads, 64).permute(2, 0, 3, 1, 4)
    mask = torch.full((L, L), float("-inf"), device="cuda").triu_(1)
    s = r16(r16(q * 0.125) @ k.transpose(-1, -2)) + mask
    p = r16(torch.softmax(s, dim=-1))
    ref = r16(p @ v).transpose(1, 2).reshape(K * L, D)
    diff = (got - ref).abs()
    ulp = torch.maximum(ref.abs(), torch.tensor(2.0 ** -14, device="cuda")).log2().floor().exp2() * 2.0 ** -10
    assert (diff <= 2 * ulp).all(), f"text_attn: {int((diff > 2 * ulp).sum())} elements off by more than 2 fp16 ulp"
    frac_exact = (diff == 0).float().mean().item()
    assert frac_exact > 0.97, f"text_attn: only {frac_exact:.4f} of the outputs bit-identical to the fp16-step recipe"
    # and it agrees with the flash kernel to fp16 accuracy (different rounding points, same function)
    _close(ops.mhsa(qkv, K, L, heads, True), ref, 3e-3, "mhsa vs fp16-step recipe")


def test_layernorm(ops):
    for dtype, C, eps in [(torch.float32, 1024, 1e-6), (torch.float16, 512, 1e-5)]:
        x = _rand((777, C), 20, 3.0, dtype) + 0.5
        g = _rand((C,), 21, 1.0, torch.float32)
        b = _rand((C,), 22, 1.0, torch.float32)
        y = ops.layernorm(x, g, b, eps)
        _close(y, F.layer_norm(x.float(), (C,), g, b, eps), 1e-3, f"layernorm {dtype}")


def test_patch_tokens_pos(ops):
    B, H, W = 2, 64, 96
    x = _rand((B, 3, H, W), 23, 1.0, torch.float32).clamp(-1, 1)
    a = ops.patchify(x)
    ref = F.unfold(x, 16, stride=16).transpose(1, 2).reshape(B * 24, 768)
    _close(a, ref, 1e-3, "patchify")
    pos = _rand((1 + 24 * 24, 1024), 24, 0.02, torch.float32)
    pr = ops.pos_resize(pos, 24, 4, 6)
    grid = pos[1:].view(1, 24, 24, 1024).permute(0, 3, 1, 2)
    refp = F.interpolate(grid, size=(4, 6), mode="bilinear").permute(0, 2, 3, 1).reshape(24, 1024)
    _close(pr[1:], refp, 1e-5, "pos resize")
    _close(pr[:1], pos[:1], 0, "pos cls")
    patch = _rand((B * 24, 1024), 25, 1.0, torch.float32)
    cls = _rand((1024,), 26, 1.0, torch.float32)
    xt = ops.assemble_tokens(patch, cls, pr, B, 24)
    reft = torch.cat([cls.view(1, 1, -1).expand(B, -1, -1), patch.view(B, 24, 1024)], 1) + pr
    _close(xt, reft, 1e-6, "assemble")
    tok, c16 = ops.readout_split(xt)
    _close(tok, xt[:, 1:].reshape(B * 24, 1024), 1e-3, "readout tok")
    _close(c16[:B], xt[:, 0], 1e-3, "readout cls")


def test_im2col_upsample_norms(ops):
    x = _rand((2, 30, 30, 64), 27)
    a = ops.im2col_3x3_s2(x)
    cols = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1, stride=2)  # [B, C*9, L], index c*9+tap
    ref = cols.view(2, 64, 9, 225).permute(0, 3, 2, 1).reshape(2 * 225, 9 * 64)
    _close(a, ref, 0, "im2col s2")
    y = ops.upsample2x_nhwc(x)
    refu = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    _close(y, refu.permute(0, 2, 3, 1), 1e-3, "upsample nhwc")
    for shape in ((2, 15, 15, 256), (1, 30, 41, 256), (3, 7, 60, 256)):  # fp32 input (after out_conv), odd widths
        xf = _rand(shape, 27, 2.0, torch.float32)
        want = F.interpolate(xf.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
        _close(ops.upsample2x_nhwc(xf, torch.float32), want, 2e-6, "upsample nhwc fp32 -> fp32")
        _close(ops.upsample2x_nhwc(xf, torch.float16), want, 1e-3, "upsample nhwc fp32 -> fp16")
        skip = _rand(tuple(want.shape), 26, 1.0, torch.float32)
        _close(ops.upsample2x_nhwc(xf, torch.float32, add=skip), want + skip, 2e-6, "upsample nhwc fp32 + skip")
        xh = xf.half()  # the engine's variant: fp16 source (low-res out_conv result)
        wanth = F.interpolate(xh.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear",
                              align_corners=True).permute(0, 2, 3, 1)
        _close(ops.upsample2x_nhwc(xh, torch.float32, add=skip), wanth + skip, 2e-6, "upsample nhwc fp16 -> fp32 + skip")
        _close(ops.upsample2x_nhwc(xh, torch.float16, decoder=True), wanth, 1e-3, "upsample nhwc fp16 -> fp16 (decoder)")
    lg = _rand((2, 5, 24, 40), 28, 3.0)
    up = ops.upsample2x_nchw(lg)
    _close(up, F.interpolate(lg.float(), scale_factor=2, mode="bilinear", align_corners=True), 1e-6, "upsample nchw")
    f = _rand((1000, 512), 29, 2.0, torch.float32)
    ls = math.exp(math.log(1 / 0.07))
    n16 = ops.l2norm_scale(f, ls)
    refn = (torch.tensor(ls) * (f / f.norm(dim=-1, keepdim=True)).half()).float()
    _close(n16, refn, 1e-3, "l2norm_scale")
    t = _rand((150, 512), 30, 0.3)
    tn = ops.l2norm_f16(t)
    _close(tn, (t / t.norm(dim=-1, keepdim=True)).float(), 1e-3, "l2norm f16")


@pytest.mark.parametrize("B,K,H,W", [(2, 5, 24, 40), (1, 150, 40, 40), (1, 2, 16, 8), (1, 7, 8, 264)])
def test_upsample_argmax_matches_logits(ops, B, K, H, W):
    """SURVEY 8(f) row 2: the fused upsample+argmax returns torch.max(logits, 1)[1] of the logits the unfused path
    produces — same interpolated values bit for bit, first maximal class on ties (ties are provoked: fp16 inputs on a
    coarse grid, duplicated class planes)."""
    lg = (_rand((B, K, H, W), 31, 2.0) * 4).round() / 4  # coarse values -> many exact ties after interpolation
    if K > 3:
        lg[:, 3] = lg[:, 1]  # an exactly duplicated class: the first index must win
    up = ops.upsample2x_nchw(lg)
    m = ops.upsample2x_argmax(lg)
    assert m.dtype == torch.int64 and m.shape == (B, 2 * H, 2 * W)
    assert torch.equal(m, up.argmax(1)) or torch.equal(up.gather(1, m[:, None]), up.max(1, keepdim=True)[0])
    # first-maximum rule (what torch.max returns on CPU)
    assert torch.equal(m.cpu(), torch.max(up.cpu(), 1)[1])
    # the shared-memory-free kernel of the multi-GPU gather: the same values bit for bit
    assert torch.equal(ops.upsample2x_nchw(lg, background=True), up)


@pytest.mark.parametrize("mode,act,in_f16", [(1, "lrelu", True), (1, "none", False), (2, "tanh", True), (2, "relu", False)])
def test_head_block(ops, mode, act, in_f16):
    """scratch.head_block (arch_option 1 = bottleneck_block, 2 = depthwise_block; lseg_net.py:29-79): one shared 3x3 kernel
    over every class plane, optional channel-max skip, optional activation — against torch's own conv2d / max."""
    from lseg_b200 import _lib
    B, K, h, w = 2, 7, 37, 56
    x = _rand((B, K, h, w), 61, 1.5, torch.float16 if in_f16 else torch.float32)
    wt = _rand((1, 1, 3, 3), 62, 0.3, torch.float32)
    bias = 0.17
    got = ops.head_block(x, wt.flatten().tolist(), bias, mode, _lib.HEAD_ACT[act])
    xf = x.float()
    ref = F.conv2d(xf.reshape(-1, 1, h, w), wt, torch.tensor([bias], device="cuda"), padding=1).view(B, K, h, w)
    if mode == 1:
        ref = ref + xf.max(dim=1, keepdim=True)[0]
    ref = {"none": lambda t: t, "relu": F.relu, "lrelu": lambda t: F.leaky_relu(t, 0.01), "tanh": torch.tanh}[act](ref)
    _close(got, ref, 2e-6, f"head_block mode {mode} {act}")
    up = ops.upsample2x_nchw_f32(got)
    _close(up, F.interpolate(got, scale_factor=2, mode="bilinear", align_corners=True), 1e-6, "fp32-input upsample")


def test_text_glue(ops):
    K, L, Wd = 5, 77, 512
    g = torch.Generator().manual_seed(31)
    tokens = torch.zeros((K, L), dtype=torch.int64)
    for k in range(K):
        n = 1 + k
        tokens[k, 0] = 49406
        tokens[k, 1:1 + n] = torch.randint(1000, 40000, (n,), generator=g)
        tokens[k, 1 + n] = 49407
    tokens = tokens.cuda()
    emb = _rand((49408, Wd), 32, 0.02, torch.float32)
    pos = _rand((L, Wd), 33, 0.01, torch.float32)
    x = ops.text_embed(tokens, emb, pos)
    ref = (emb[tokens].half() + pos.half()).view(K * L, Wd)
    _close(x, ref.float(), 0, "text embed")
    eot = ops.text_eot_gather(tokens, x)
    _close(eot[:K], x.view(K, L, Wd)[torch.arange(K), tokens.argmax(-1)].float(), 0, "eot gather")
