"""The GEMM's tile schedule must not change results: each persistent CTA deals its work list out to two consumer
warpgroups in turn, so which warpgroup computes a tile depends on the grid and on the tile's place in the list. These
tests compute the same output tiles under different schedules (a 128-row slice alone vs inside the full GEMM, one image
vs a batch) and require bit-identical results, on shapes that give CTAs odd tile counts, grids smaller than the SM
count, M tails, every epilogue mode and the fixed split-K schedule.
"""
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


def _run_linear(ops, mode, a_pad, w, M, N, bias, scale, res):
    """One GEMM in the given epilogue mode; returns its outputs."""
    dev = "cuda"
    if mode == "tma_f16":
        o16 = torch.zeros((M, N), dtype=torch.float16, device=dev)
        ops.gemm(a_pad, w, N, M=M, bias=bias, act=ops.ACT_GELU, out_f16=o16)
        return [o16]
    if mode == "tma_add":
        x = res.clone()
        ops.gemm(a_pad, w, N, M=M, bias=bias, res_f32=x, out_f32=x)
        return [x]
    if mode == "direct":
        o32 = torch.zeros((M, N), dtype=torch.float32, device=dev)
        r16 = torch.zeros((M, N), dtype=torch.float16, device=dev)
        ops.gemm(a_pad, w, N, M=M, bias=bias, scale=scale, res_f32=res, out_f32=o32, out_f16_relu=r16)
        return [o32, r16]
    assert mode == "relu_res"
    x = res.clone()
    o16 = torch.zeros((M, N), dtype=torch.float16, device=dev)
    ops.gemm(a_pad, w, N, M=M, bias=bias, scale=scale, res_f32=x, out_f32=x, out_f16=o16, relu_after_res=True)
    return [x, o16]


# (M, N): 200 x 2 = 400 tiles on 132 SMs (most CTAs own 3 tiles, some 4; M tail of 91 rows) and 8 x 2 = 16 tiles
# (grid smaller than the SM count: every CTA owns one tile, its second warpgroup stays idle)
@pytest.mark.parametrize("M,N", [(199 * 128 + 91, 256), (7 * 128 + 100, 256)])
@pytest.mark.parametrize("mode", ["tma_f16", "tma_add", "direct", "relu_res"])
def test_gemm_slice_equals_full(ops, mode, M, N):
    K = 256
    a = _rand((M, K), 11)
    a_pad = ops.pad_rows(a)
    w = ops.pad_rows(_rand((N, K), 12, 0.05))
    bias = _rand((N,), 13, 1.0, torch.float32)
    scale = _rand((N,), 14, 0.5, torch.float32).abs() + 0.5
    res = _rand((M, N), 15, 1.0, torch.float32)
    full = _run_linear(ops, mode, a_pad, w, M, N, bias, scale, res)

    pre = a.float() @ w[:N].float().t()
    if mode == "tma_f16":
        ref = F.gelu(pre + bias)
    elif mode == "tma_add":
        ref = res + pre + bias
    elif mode == "direct":
        ref = res + pre * scale + bias
    else:
        ref = torch.relu(res + pre * scale + bias)
    err = (full[0].float() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 2e-3, f"{mode}: max rel err {err:.3e} against the fp32 reference"

    m_tiles = (M + 127) // 128
    for t in sorted({0, min(137, m_tiles - 1), m_tiles - 1}):  # first tile, one past the first wave, the M tail
        r0 = t * 128
        rows = min(128, M - r0)
        part = _run_linear(ops, mode, a_pad[r0:r0 + 128], w, rows, N, bias, scale, res[r0:r0 + rows].contiguous())
        for got, want in zip(part, full):
            assert torch.equal(got, want[r0:r0 + rows]), f"{mode}: rows {r0}..{r0 + rows} differ from the full GEMM"


def _conv(ops, kind, x, w, sc, sh, res):
    B, H, W, _ = x.shape
    P = B * H * W
    dev = "cuda"
    if kind == "conv_f16":  # RCU conv1: folded BN + ReLU, fp16 out (TMA store)
        o = torch.zeros((P, 256), dtype=torch.float16, device=dev)
        ops.gemm(x, w, 256, conv=(3, 1), scale=sc, bias=sh, act=ops.ACT_RELU, out_f16=o, ldc=256)
        return [o]
    o32 = torch.zeros((P, 256), dtype=torch.float32, device=dev)
    r16 = torch.zeros((P, 256), dtype=torch.float16, device=dev)
    ops.gemm(x, w, 256, conv=(3, 1), scale=sc, bias=sh, res_f32=res, out_f32=o32, out_f16_relu=r16, ldc=256)
    return [o32, r16]  # RCU conv2: register-direct; on the 15 x 15 level also the fixed split-K schedule


# 30 x 30, B = 20: 8 x 2 tiles per image, 320 tiles -> 2 or 3 per CTA. 15 x 15, B = 20: the fixed split-K schedule
# (4 segments per tile, sized for 8 images) -> 320 units -> 2 or 3 per CTA; one image alone runs 16 units on 16 CTAs.
@pytest.mark.parametrize("side,kind", [(30, "conv_f16"), (30, "conv_direct"), (15, "conv_direct")])
def test_conv_image_equals_batch(ops, side, kind):
    B = 20
    x = _rand((B, side, side, 256), 21)
    w = ops.pad_rows(_rand((256, 9 * 256), 22, 0.02))
    sc = _rand((256,), 23, 0.5, torch.float32).abs() + 0.5
    sh = _rand((256,), 24, 1.0, torch.float32)
    res = _rand((B * side * side, 256), 25, 1.0, torch.float32)
    full = _conv(ops, kind, x, w, sc, sh, res)

    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False  # an fp32 reference, not a TF32 one
    try:
        ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w[:256].float().view(256, 3, 3, 256).permute(0, 3, 1, 2),
                       padding=1)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    ref = ref.permute(0, 2, 3, 1).reshape(-1, 256) * sc + sh
    ref = torch.relu(ref) if kind == "conv_f16" else ref + res
    err = (full[0].float() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 2e-3, f"{kind} {side}: max rel err {err:.3e} against the fp32 reference"

    P = side * side
    for b in (0, 7, B - 1):
        one = _conv(ops, kind, x[b:b + 1].contiguous(), w, sc, sh, res[b * P:(b + 1) * P].contiguous())
        for got, want in zip(one, full):
            assert torch.equal(got, want[b * P:(b + 1) * P]), f"{kind} {side}: image {b} alone differs from the batch"
