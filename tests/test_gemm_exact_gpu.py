"""Every GEMM planner path against an exact oracle, with guard bands around every output.

Operands are small integers (A in -2..2, W in -1..1, K_total <= 9216), so every partial sum is an integer below 2^15 and
the fp32 accumulation is exact in any order and under any split: tensor-core accumulation, TMA reduce-add, stream-K and
the fixed split-K reduce. Scales are powers of two, biases and fp32 residuals multiples of 0.25 in [-8, 8], fp16 residuals
small integers. Every fp32 output must therefore equal a float64 reference exactly, and every fp16 output must equal that
reference rounded once to fp16: a difference is a wrong tile, a wrong k-chunk count or a wrong mapping, never rounding.
The activations GELU and QuickGELU are the exceptions; they are checked against their documented error bounds.

Each output lives inside a larger buffer filled with a NaN sentinel (or, for an in-place residual, with the residual
itself); everything outside the M x N window must keep its bits. Each case also asserts, through lseg_debug_gemm_plan,
the plan it is meant to exercise, so a planner change or another SM count cannot move it off its path silently.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# lseg_debug_gemm_plan: epilogue kinds and kernel instantiations
EPI_DIRECT, EPI_TMA_F16, EPI_TMA_ADD = 0, 1, 2
K_DIRECT, K_TMA_F16, K_TMA_ADD, K_FIXED_SPLIT, K_GROUPED, K_RELU_RES = 0, 1, 2, 3, 4, 5
SENTINEL = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7E5A}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16}


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


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def nondeterministic(ops):
    ops.set_deterministic(False)
    try:
        yield
    finally:
        ops.set_deterministic(True)


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _ints(shape, lo, hi, seed, dtype=torch.float16):
    return torch.randint(lo, hi + 1, shape, generator=_gen(seed)).to(dtype).cuda()


def _quarters(shape, seed):  # multiples of 0.25 in [-8, 8]
    return (torch.randint(-32, 33, shape, generator=_gen(seed)).float() * 0.25).cuda()


def _pow2(shape, seed):  # 0.5, 1 or 2
    return (2.0 ** torch.randint(-1, 2, shape, generator=_gen(seed)).float()).cuda()


def _operands(M, N, K, seed, a_rows=None):
    """A [a_rows >= max(M, 128), K] (rows beyond M hold data too: they must not reach the output), W [rows padded, K]."""
    a = _ints((a_rows or max(M, 128), K), -2, 2, seed)
    w = _ints((N, K), -1, 1, seed + 1)
    return a, w


def _guarded(M, ldc, dtype, fill=None):
    """[M + 2, ldc] buffer of sentinel bits (or `fill`); returns (buffer, view of rows 1 .. M)."""
    if fill is None:
        buf = torch.full((M + 2, ldc), SENTINEL[dtype], dtype=BITS[dtype], device="cuda").view(dtype)
    else:
        buf = fill.clone()
    return buf, buf[1:M + 1]


def _flat(n, dtype, guard=8):
    """Flat buffer with `guard` sentinel elements before and after; returns (buffer, view of the n inner elements)."""
    buf = torch.full((n + 2 * guard,), SENTINEL[dtype], dtype=BITS[dtype], device="cuda").view(dtype)
    return buf, buf[guard:guard + n]


def _untouched(before, after, keep, what):
    """Every element where `keep` is True still holds its bits."""
    b, a = before.view(BITS[before.dtype]), after.view(BITS[after.dtype])
    bad = int(((a != b) & keep).sum())
    assert bad == 0, f"{what}: {bad} elements outside the output window were written"


def _window_mask(buf, M, N):
    keep = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    keep[1:M + 1, :N] = False
    return keep


def _exact(got, ref, what):
    """got (fp32 / fp16) equals the float64 reference rounded once to got's type."""
    want = ref.to(got.dtype)
    assert not torch.isnan(got).any(), f"{what}: NaN in the output window (unwritten sentinel?)"
    bad = got != want
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {n} of {got.numel()} elements differ; first at {idx}: "
                             f"got {got[tuple(idx)].item()}, want {want[tuple(idx)].item()}")


def _plan(ops, want, what, **plan):
    got = ops.gemm_plan(**plan)
    for k, v in want.items():
        assert got[k] == v, f"{what}: plan {got}, expected {k} = {v}"
    return got


def _mm(a, w, M, N):
    return a[:M].double() @ w[:N].double().t()


# ---------------------------------------------------------------------------------------------------------------------
# plain linears, one shape list through each epilogue kind
# ---------------------------------------------------------------------------------------------------------------------
def _plain_shapes(sms):
    return [
        (1, 64, 64), (127, 2, 64), (128, 8, 192), (129, 24, 1024), (sms * 128, 128, 192),  # tiles == SMs
        (sms * 128 + 1, 72, 64),  # SMs + 1 tiles, a 64-column TMA tile plus an 8-column tail
        (7208, 1024, 1024), (1808, 3072, 2112),  # ViT-L/16 at 480^2 (B = 8); 33 k-chunks
        (300, 56, 4096), (300, 136, 1024), (1808, 200, 64), (1000, 150, 1024)]


PLAIN = [(i, mode) for i in range(12) for mode in ("tma_f16", "tma_add", "direct", "relu_res")]


@pytest.mark.parametrize("idx,mode", PLAIN)
def test_plain(ops, sms, idx, mode):
    M, N, K = _plain_shapes(sms)[idx]
    ldc = (N + 8 + 7) // 8 * 8  # ldc > N
    a, w = _operands(M, N, K, 100 + idx, a_rows=None if idx % 2 else max(M + 37, 128))
    wp = ops.pad_rows(w)
    bias = _quarters((N,), 200 + idx)
    scale = _pow2((N,), 300 + idx)
    acc = _mm(a, w, M, N)
    tma_ok = N % 8 == 0 and N >= 64
    what = f"{mode} M={M} N={N} K={K}"
    if mode == "tma_f16":
        buf, out = _guarded(M, ldc, torch.float16)
        kw = dict(bias=bias, act=ops.ACT_RELU, out_f16=out, ldc=ldc, M=M)
        _plan(ops, {"kernel": K_TMA_F16 if tma_ok else K_DIRECT, "split_fixed": 0}, what, a=a, w=wp, N=N, **kw)
        before = buf.clone()
        ops.gemm(a, wp, N, **kw)
        _exact(out[:, :N], (acc + bias.double()).clamp_min(0), what)
        _untouched(before, buf, _window_mask(buf, M, N), what)
    elif mode == "tma_add":
        res = _quarters((M + 2, ldc), 400 + idx)
        buf, x = _guarded(M, ldc, torch.float32, fill=res)
        kw = dict(bias=bias, res_f32=x, out_f32=x, ldc=ldc, M=M)
        _plan(ops, {"kernel": K_TMA_ADD if tma_ok else K_DIRECT, "split_k": 0}, what, a=a, w=wp, N=N, **kw)
        before = buf.clone()
        ops.gemm(a, wp, N, **kw)
        _exact(x[:, :N], res[1:M + 1, :N].double() + acc + bias.double(), what)
        _untouched(before, buf, _window_mask(buf, M, N), what)
    else:
        res = _quarters((M, ldc), 500 + idx)
        b32, o32 = _guarded(M, ldc, torch.float32)
        b16, o16 = _guarded(M, ldc, torch.float16)
        kw = dict(bias=bias, scale=scale, res_f32=res, out_f32=o32, out_f16=o16, ldc=ldc, M=M)
        ref = acc * scale.double() + bias.double() + res[:, :N].double()
        if mode == "relu_res":
            kw["relu_after_res"] = True
            ref = ref.clamp_min(0)
        _plan(ops, {"kernel": K_RELU_RES if mode == "relu_res" else K_DIRECT, "epi": EPI_DIRECT}, what,
              a=a, w=wp, N=N, **kw)
        before32, before16 = b32.clone(), b16.clone()
        ops.gemm(a, wp, N, **kw)
        _exact(o32[:, :N], ref, what + " fp32")
        _exact(o16[:, :N], ref.float(), what + " fp16")
        _untouched(before32, b32, _window_mask(b32, M, N), what + " fp32")
        _untouched(before16, b16, _window_mask(b16, M, N), what + " fp16")


# ---------------------------------------------------------------------------------------------------------------------
# epilogue options
# ---------------------------------------------------------------------------------------------------------------------
def test_every_direct_output(ops):
    """scale, bias, two fp32 residuals, fp32 + fp16 + relu-fp16 outputs in one call; then the fp16 residual stream."""
    M, N, K, ldc = 1000, 200, 1024, 216
    a, w = _operands(M, N, K, 1)
    wp = ops.pad_rows(w)
    bias, scale = _quarters((N,), 2), _pow2((N,), 3)
    r1, r2 = _quarters((M, ldc), 4), _quarters((M, ldc), 5)
    bufs = {k: _guarded(M, ldc, dt) for k, dt in (("o32", torch.float32), ("o16", torch.float16),
                                                  ("orl", torch.float16))}
    before = {k: b.clone() for k, (b, _) in bufs.items()}
    kw = dict(bias=bias, scale=scale, res_f32=r1, res2_f32=r2, out_f32=bufs["o32"][1], out_f16=bufs["o16"][1],
              out_f16_relu=bufs["orl"][1], ldc=ldc)
    _plan(ops, {"kernel": K_DIRECT}, "all outputs", a=a, w=wp, N=N, **kw)
    ops.gemm(a, wp, N, **kw)
    ref = _mm(a, w, M, N) * scale.double() + bias.double() + r1[:, :N].double() + r2[:, :N].double()
    _exact(bufs["o32"][1][:, :N], ref, "fp32")
    _exact(bufs["o16"][1][:, :N], ref.float(), "fp16")
    _exact(bufs["orl"][1][:, :N], ref.clamp_min(0).float(), "relu fp16")
    for k, (b, _) in bufs.items():
        _untouched(before[k], b, _window_mask(b, M, N), k)
    # fp16 residual: the branch output is rounded to fp16 first, then added in fp16 (rounded once more)
    r16 = _ints((M, ldc), -4, 4, 6)
    b16, o16 = _guarded(M, ldc, torch.float16)
    before16 = b16.clone()
    kw = dict(bias=bias, res_f16=r16, out_f16=o16, ldc=ldc)
    _plan(ops, {"kernel": K_DIRECT}, "fp16 residual", a=a, w=wp, N=N, **kw)
    ops.gemm(a, wp, N, **kw)
    branch = (_mm(a, w, M, N) + bias.double()).half()
    _exact(o16[:, :N], (branch.double() + r16[:, :N].double()).float(), "fp16 residual")
    _untouched(before16, b16, _window_mask(b16, M, N), "fp16 residual")


@pytest.mark.parametrize("N,tma", [(512, True), (512, False), (200, False)])
def test_out_row_sumsq(ops, N, tma):
    """Partial squared row norms per 32-column chunk (K = 64 keeps every square and sum exact), on the TMA fp16 path
    (head1) and the register-direct path, with a 200-column output whose last chunk is partial."""
    M, K = 1000, 64
    parts = (N + 31) // 32
    a, w = _operands(M, N, K, 7)
    wp = ops.pad_rows(w)
    bias = _quarters((N,), 8)
    sbuf, ss = _flat(M * parts, torch.float32)
    b16, o16 = _guarded(M, N, torch.float16)
    kw = dict(bias=bias, out_f16=o16[:, :N], out_row_sumsq=ss.view(M, parts))
    if not tma:  # an fp32 output as well: the register-direct epilogue
        b32, o32 = _guarded(M, N, torch.float32)
        kw["out_f32"] = o32
    _plan(ops, {"kernel": K_TMA_F16 if tma else K_DIRECT}, f"sumsq N={N}", a=a, w=wp, N=N, **kw)
    before, before16 = sbuf.clone(), b16.clone()
    ops.gemm(a, wp, N, **kw)
    x = _mm(a, w, M, N) + bias.double()
    ref = F.pad(x * x, (0, parts * 32 - N)).view(M, parts, 32).sum(-1)
    _exact(ss.view(M, parts), ref, "row sumsq")
    _exact(o16, x.float(), "fp16 out")
    if not tma:
        _exact(o32, x, "fp32 out")
    keep = torch.ones_like(sbuf, dtype=torch.bool)
    keep[8:8 + M * parts] = False
    _untouched(before, sbuf, keep, "row sumsq")
    _untouched(before16, b16, _window_mask(b16, M, N), "fp16 out")


def _gelu64(x):
    return x * 0.5 * torch.special.erfc(-x / math.sqrt(2.0))


def _ulp16(v):
    """fp16 ulp at |v| (the subnormal spacing 2^-24 below 2^-14)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _check_gelu(got, pre, what):
    """GELU(erf) of the exact pre-activation: fp32 within the documented 3.7e-6 (common.cuh gelu_erf) plus 2^-21 |x| for
    the final fp32 product; fp16 within 1 ulp, or within that fp32 bound plus the fp16 rounding (half an ulp) where that
    is more: below |gelu| = 2^-7 an fp16 ulp is smaller than twice the fp32 error bound."""
    ref = _gelu64(pre)
    g = got.double()
    err = (g - ref).abs()
    tol = 3.7e-6 + 2.0 ** -21 * pre.abs()
    if got.dtype == torch.float16:  # the fp16 result is the fp32 one rounded once
        ulp = _ulp16(ref)
        tol = torch.maximum(ulp, tol + 0.5 * ulp)
        inf = torch.isinf(ref.half())
        assert torch.equal(got[inf], ref.half()[inf]), f"{what}: overflow to fp16 inf differs"
        err, tol = err[~inf], tol[~inf]
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} values off; worst excess {float((err - tol).max()):.3e}"


@pytest.mark.parametrize("group_rows,B", [(900, 3), (225, 8)])
@pytest.mark.parametrize("path", ["direct", "tma_gelu"])
def test_grouped_bias(ops, group_rows, B, path):
    """Per-image bias rows (the readout's T at 480^2: 900 for ViT-L/16, 225 for ViT-B/32): groups straddle tiles."""
    M, N, K = group_rows * B, 1024, 192
    a, w = _operands(M, N, K, 9)
    wp = ops.pad_rows(w)
    gb = _quarters((B, N), 10)
    pre = _mm(a, w, M, N) + gb.double().repeat_interleave(group_rows, 0)
    if path == "direct":
        buf, out = _guarded(M, N, torch.float32)
        kw = dict(bias=gb, bias_group_rows=group_rows, out_f32=out)
        want = K_DIRECT
    else:
        buf, out = _guarded(M, N, torch.float16)
        kw = dict(bias=gb, bias_group_rows=group_rows, act=ops.ACT_GELU, out_f16=out)
        want = K_TMA_F16
    _plan(ops, {"kernel": want}, path, a=a, w=wp, N=N, **kw)
    before = buf.clone()
    ops.gemm(a, wp, N, **kw)
    if path == "direct":
        _exact(out, pre, "grouped bias")
    else:
        _check_gelu(out, pre, "grouped bias + gelu")
    _untouched(before, buf, _window_mask(buf, M, N), path)


def test_n150_grouped_bias(ops):
    """N % 4 != 0 with a grouped bias: bias row g starts at g * 150 floats, not 16-byte aligned for odd g."""
    M, N, K, G = 1000, 150, 64, 250
    a, w = _operands(M, N, K, 11)
    wp = ops.pad_rows(w)
    gb = _quarters((M // G, N), 12)
    buf, out = _guarded(M, 152, torch.float32)
    kw = dict(bias=gb, bias_group_rows=G, out_f32=out, ldc=152)
    _plan(ops, {"kernel": K_DIRECT}, "n150", a=a, w=wp, N=N, **kw)
    before = buf.clone()
    ops.gemm(a, wp, N, **kw)
    _exact(out[:, :N], _mm(a, w, M, N) + gb.double().repeat_interleave(G, 0), "N=150 grouped bias")
    _untouched(before, buf, _window_mask(buf, M, N), "N=150 grouped bias")


# ---------------------------------------------------------------------------------------------------------------------
# implicit-GEMM convs
# ---------------------------------------------------------------------------------------------------------------------
def _conv_ref(x, w, N, ksize, pad):
    B, H, W, C = x.shape
    wt = w[:N].double().view(N, ksize, ksize, C).permute(0, 3, 1, 2)
    y = F.conv2d(x.double().permute(0, 3, 1, 2), wt, padding=pad)
    return y.permute(0, 2, 3, 1).reshape(B * H * W, N)


def _fixed_split(sms, H, W, N, k_iters, tma_f16):
    """gemm_pick_split's segment count for a plain-epilogue conv (lang-seg_b200/csrc/lseg_b200.cu)."""
    ref_tiles = 8 * ((H + 7) // 8) * ((W + 15) // 16) * ((N + 127) // 128)
    if ref_tiles * 2 > sms:
        return 0
    s = min(sms // ref_tiles, k_iters // 4, 16)
    if s < 4 and tma_f16:
        return 0
    return s if s >= 2 else 0


CONVS = [  # B, H, W, Cin, N, (ksize, pad)
    (2, 1, 1, 64, 64, (3, 1)), (1, 3, 5, 256, 128, (1, 0)), (2, 8, 16, 64, 192, (3, 1)), (1, 9, 17, 1024, 256, (3, 1)),
    (3, 15, 15, 256, 64, (1, 0)), (1, 17, 33, 64, 128, (3, 1)), (2, 30, 30, 256, 256, (3, 1)),
    (2, 30, 30, 1024, 128, (1, 0))]


@pytest.mark.parametrize("idx", range(len(CONVS)))
@pytest.mark.parametrize("mode", ["tma_f16", "direct"])
def test_conv(ops, sms, idx, mode):
    B, H, W, Cin, N, conv = CONVS[idx]
    P = B * H * W
    ldc = N + 64
    x = _ints((B, H, W, Cin), -2, 2, 20 + idx)
    w = _ints((N, conv[0] * conv[0] * Cin), -1, 1, 40 + idx)
    wp = ops.pad_rows(w)
    scale, bias = _pow2((N,), 60 + idx), _quarters((N,), 80 + idx)
    acc = _conv_ref(x, w, N, *conv)
    k_iters = conv[0] * conv[0] * Cin // 64
    what = f"conv {mode} {B}x{H}x{W}x{Cin} -> {N} k{conv[0]}"
    if mode == "tma_f16":
        buf, out = _guarded(P, ldc, torch.float16)
        kw = dict(conv=conv, scale=scale, bias=bias, act=ops.ACT_RELU, out_f16=out, ldc=ldc)
        split = _fixed_split(sms, H, W, N, k_iters, True)
        ref = (acc * scale.double() + bias.double()).clamp_min(0)
        outs = [(buf, out)]
    else:
        res = _quarters((P, ldc), 100 + idx)
        b32, o32 = _guarded(P, ldc, torch.float32)
        b16, orl = _guarded(P, ldc, torch.float16)
        kw = dict(conv=conv, scale=scale, bias=bias, res_f32=res, out_f32=o32, out_f16_relu=orl, ldc=ldc)
        split = _fixed_split(sms, H, W, N, k_iters, False)
        ref = acc * scale.double() + bias.double() + res[:, :N].double()
        outs = [(b32, o32), (b16, orl)]
    want = {"split_fixed": split, "kernel": K_FIXED_SPLIT if split else (K_TMA_F16 if mode == "tma_f16" else K_DIRECT)}
    _plan(ops, want, what, a=x, w=wp, N=N, **kw)
    before = [b.clone() for b, _ in outs]
    ops.gemm(x, wp, N, **kw)
    if mode == "tma_f16":
        _exact(out[:, :N], ref.float(), what)
    else:
        _exact(o32[:, :N], ref, what + " fp32")
        _exact(orl[:, :N], ref.clamp_min(0).float(), what + " relu fp16")
    for (b, _), b0 in zip(outs, before):
        _untouched(b0, b, _window_mask(b, P, N), what)


def _split_geometry(sms, target):
    """A (B, H, W, Cin, N) whose fixed split-K segment count is `target` (None: the planner's maximum)."""
    cands = [(2, 8, 16, 1024, 128), (8, 15, 15, 256, 256), (8, 15, 15, 1024, 128), (8, 17, 17, 256, 128),
             (4, 17, 33, 256, 128), (8, 30, 30, 256, 128), (2, 8, 16, 256, 256), (3, 8, 16, 256, 384)]
    splits = {c: _fixed_split(sms, c[1], c[2], c[4], 9 * c[3] // 64, False) for c in cands}
    target = max(splits.values()) if target is None else target
    for c, s in splits.items():
        if s == target:
            return c, s
    pytest.skip(f"no candidate geometry gives {target} split-K segments on {sms} SMs")


@pytest.mark.parametrize("target", [2, 4, None])
@pytest.mark.parametrize("epi", ["rcu", "relu_res", "gelu", "quickgelu", "relu"])
def test_conv_fixed_split(ops, sms, target, epi):
    """Deterministic split-K: raw partials per segment, then splitk_reduce_kernel applies the epilogue (ldc > N)."""
    (B, H, W, Cin, N), split = _split_geometry(sms, target)
    P, ldc = B * H * W, N + 32
    x = _ints((B, H, W, Cin), -2, 2, 130)
    w = _ints((N, 9 * Cin), -1, 1, 131)
    wp = ops.pad_rows(w)
    scale, bias = _pow2((N,), 132), _quarters((N,), 133)
    r1, r2 = _quarters((P, ldc), 134), _quarters((P, ldc), 135)
    pre = _conv_ref(x, w, N, 3, 1) * scale.double() + bias.double()
    b32, o32 = _guarded(P, ldc, torch.float32)
    b16, o16 = _guarded(P, ldc, torch.float16)
    brl, orl = _guarded(P, ldc, torch.float16)
    kw = dict(conv=(3, 1), scale=scale, bias=bias, out_f32=o32, ldc=ldc)
    if epi == "rcu":
        kw.update(res_f32=r1, res2_f32=r2, out_f16=o16, out_f16_relu=orl)
        ref = pre + r1[:, :N].double() + r2[:, :N].double()
    elif epi == "relu_res":
        kw.update(res_f32=r1, out_f16=o16, relu_after_res=True)
        ref = (pre + r1[:, :N].double()).clamp_min(0)
    else:
        kw.update(act={"gelu": ops.ACT_GELU, "quickgelu": ops.ACT_QUICKGELU, "relu": ops.ACT_RELU}[epi], out_f16=o16)
        ref = pre.clamp_min(0) if epi == "relu" else None
    what = f"split-K {split} {epi} {B}x{H}x{W}x{Cin} -> {N}"
    _plan(ops, {"split_fixed": split, "kernel": K_FIXED_SPLIT, "epi": EPI_DIRECT}, what, a=x, w=wp, N=N, **kw)
    before = [b.clone() for b in (b32, b16, brl)]
    ops.gemm(x, wp, N, **kw)
    if epi == "gelu":
        _check_gelu(o32[:, :N], pre, what + " fp32")
        _check_gelu(o16[:, :N], pre, what + " fp16")
    elif epi == "quickgelu":
        h = pre.half()
        q = (h * torch.sigmoid(1.702 * h)).double()
        for got in (o32[:, :N], o16[:, :N]):
            assert ((got.double() - q).abs() <= _ulp16(q)).all(), what
    else:
        _exact(o32[:, :N], ref, what + " fp32")
        _exact(o16[:, :N], ref.float(), what + " fp16")
        if epi == "rcu":
            _exact(orl[:, :N], ref.clamp_min(0).float(), what + " relu fp16")
    for b, b0 in zip((b32, b16), before):
        _untouched(b0, b, _window_mask(b, P, N), what)
    keep = _window_mask(brl, P, N) if epi == "rcu" else torch.ones_like(brl, dtype=torch.bool)  # relu copy: rcu only
    _untouched(before[2], brl, keep, what)


# ---------------------------------------------------------------------------------------------------------------------
# stream-K split of the in-place reduce-add epilogue (determinism off)
# ---------------------------------------------------------------------------------------------------------------------
def _inplace(ops, a, wp, M, N, ldc, res, **kw):
    buf, x = _guarded(M, ldc, torch.float32, fill=res)
    plan = ops.gemm_plan(a, wp, N, M=M, res_f32=x, out_f32=x, ldc=ldc, **kw)
    ops.gemm(a, wp, N, M=M, res_f32=x, out_f32=x, ldc=ldc, **kw)
    return buf, plan


@pytest.mark.parametrize("k_iters", [32, 33, 35, 64])
def test_stream_k(ops, sms, nondeterministic, k_iters):
    M, N, K, ldc = (sms + 5) * 128 - 37, 128, 64 * k_iters, 136  # SMs + 5 tiles: a ragged last wave
    a, w = _operands(M, N, K, 140 + k_iters)
    wp = ops.pad_rows(w)
    bias = _quarters((N,), 141)
    res = _quarters((M + 2, ldc), 142)
    buf, plan = _inplace(ops, a, wp, M, N, ldc, res, bias=bias)
    _exact(buf[1:M + 1, :N], res[1:M + 1, :N].double() + _mm(a, w, M, N) + bias.double(), f"stream-K k_iters={k_iters}")
    _untouched(res, buf, _window_mask(buf, M, N), "stream-K")
    assert plan["kernel"] == K_TMA_ADD and plan["split_k"] == 1, plan
    ops.set_deterministic(True)
    det, plan = _inplace(ops, a, wp, M, N, ldc, res, bias=bias)
    assert plan["split_k"] == 0, plan
    assert torch.equal(det.view(torch.int32), buf.view(torch.int32)), "stream-K result differs from the deterministic one"


def test_stream_k_off_when_tiles_divide(ops, sms, nondeterministic):
    M, N, K = 2 * sms * 128, 128, 2048
    a, w = _operands(M, N, K, 150)
    wp = ops.pad_rows(w)
    res = _quarters((M + 2, N), 151)
    buf, plan = _inplace(ops, a, wp, M, N, N, res)
    assert plan["kernel"] == K_TMA_ADD and plan["split_k"] == 0, plan
    _exact(buf[1:M + 1], res[1:M + 1].double() + _mm(a, w, M, N), "tiles % SMs == 0")


@pytest.mark.parametrize("act", ["relu", "gelu"])
def test_stream_k_inplace_activation(ops, sms, nondeterministic, act):
    """x += act(A W^T + b): the activation needs the whole K sum, so the planner must not split it."""
    M, N, K, ldc = (sms + 5) * 128 - 37, 128, 2112, 128
    a, w = _operands(M, N, K, 160)
    wp = ops.pad_rows(w)
    bias = _quarters((N,), 161)
    res = _quarters((M + 2, ldc), 162)
    code = ops.ACT_RELU if act == "relu" else ops.ACT_GELU
    buf, plan = _inplace(ops, a, wp, M, N, ldc, res, bias=bias, act=code)
    pre = _mm(a, w, M, N) + bias.double()
    r = res[1:M + 1, :N].double()
    if act == "relu":
        _exact(buf[1:M + 1, :N], r + pre.clamp_min(0), "in-place relu")
    else:  # gelu_erf's bound (see _check_gelu) plus the rounding of the fp32 residual add
        got = buf[1:M + 1, :N].double()
        tol = 3.7e-6 + 2.0 ** -21 * pre.abs() + 2.0 ** -24 * got.abs()
        assert ((got - r - _gelu64(pre)).abs() <= tol).all(), "in-place gelu"
    assert plan["kernel"] == K_TMA_ADD and plan["split_k"] == 0, plan


def test_stream_k_grouped_bias(ops, sms, nondeterministic):
    """x += A W^T + b[row / G]: the bias must be added once per tile, by the segment that starts at k = 0."""
    M, N, K, ldc, G = (sms + 5) * 128 - 37, 128, 2112, 128, 900
    a, w = _operands(M, N, K, 170)
    wp = ops.pad_rows(w)
    gb = _quarters(((M + G - 1) // G, N), 171)
    res = _quarters((M + 2, ldc), 172)
    buf, plan = _inplace(ops, a, wp, M, N, ldc, res, bias=gb, bias_group_rows=G)
    ref = res[1:M + 1, :N].double() + _mm(a, w, M, N) + gb.double().repeat_interleave(G, 0)[:M]
    _exact(buf[1:M + 1, :N], ref, "stream-K grouped bias")
    assert plan["kernel"] == K_TMA_ADD and plan["split_k"] == 1, plan


# ---------------------------------------------------------------------------------------------------------------------
# NCHW stores
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,stride,K", [(2, 2, 2), (8, 32, 30), (3, 77, 77), (5, 51, 40)])
def test_grouped_nchw(ops, B, stride, K):
    """Zero-shot label blocks: row of image b keeps columns [b*stride, b*stride + K) as channels 0..K-1. P = 900 puts image
    boundaries inside tiles; (3, 77, 77) puts image 1's block across the n-tile boundary at column 128."""
    P, D = 900, 128
    N = B * stride
    a, w = _operands(B * P, N, D, 180 + B)
    wp = ops.pad_rows(w)
    buf, out = _flat(B * K * P, torch.float16)
    kw = dict(out_f16=out.view(B, K, P), store=ops.STORE_NCHW_T, nchw=(P, K, stride))
    _plan(ops, {"kernel": K_GROUPED}, "grouped nchw", a=a, w=wp, N=N, **kw)
    before = buf.clone()
    ops.gemm(a, wp, N, **kw)
    full = _mm(a, w, B * P, N).view(B, P, N)
    ref = torch.stack([full[b, :, b * stride:b * stride + K].t() for b in range(B)])
    _exact(out.view(B, K, P), ref.float(), f"grouped nchw {B},{stride},{K}")
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[8:8 + B * K * P] = False
    _untouched(before, buf, keep, "grouped nchw")


def test_grouped_nchw_row_sumsq(ops):
    """The deferred row normalisation on the grouped store (tolerance of test_deferred_row_normalisation)."""
    B, stride, K, P, D = 3, 77, 77, 900, 512
    N = B * stride
    a, w = _operands(B * P, N, D, 190)
    wp = ops.pad_rows(w)
    sumsq = (torch.rand((B * P, D // 32), generator=_gen(191)) + 0.5).cuda()
    buf, out = _flat(B * K * P, torch.float16)
    kw = dict(out_f16=out.view(B, K, P), store=ops.STORE_NCHW_T, nchw=(P, K, stride), row_sumsq=sumsq, row_scale=14.0)
    _plan(ops, {"kernel": K_GROUPED}, "grouped nchw sumsq", a=a, w=wp, N=N, **kw)
    before = buf.clone()
    ops.gemm(a, wp, N, **kw)
    full = (_mm(a, w, B * P, N) * (14.0 / sumsq.double().sum(1, keepdim=True).sqrt())).view(B, P, N)
    ref = torch.stack([full[b, :, b * stride:b * stride + K].t() for b in range(B)])
    err = (out.view(B, K, P).double() - ref).abs().max().item() / ref.abs().max().item()
    assert err <= 2e-3, err
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[8:8 + B * K * P] = False
    _untouched(before, buf, keep, "grouped nchw sumsq")


@pytest.mark.parametrize("s,cout,g", [(8, 128, 15), (4, 192, 15), (4, 256, 30), (2, 512, 6)])
def test_depth_to_space(ops, s, cout, g):
    B, cin = 2, 128
    N = s * s * cout
    x, w = _operands(B * g * g, N, cin, 200 + s)
    wp = ops.pad_rows(w)
    bias = _quarters((cout,), 201).repeat(s * s).contiguous()
    buf, out = _flat(B * (g * s) ** 2 * cout, torch.float16)
    kw = dict(bias=bias, out_f16=out, store=ops.STORE_D2S, d2s=(s, cout, g, g), M=B * g * g)
    _plan(ops, {"kernel": K_DIRECT}, "d2s", a=x, w=wp, N=N, **kw)
    before = buf.clone()
    ops.gemm(x, wp, N, **kw)
    y = (_mm(x, w, B * g * g, N) + bias.double()).view(B, g, g, s, s, cout).permute(0, 1, 3, 2, 4, 5)
    _exact(out.view(B, g * s, g * s, cout), y.reshape(B, g * s, g * s, cout).float(), f"d2s s={s} cout={cout}")
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[8:8 + out.numel()] = False
    _untouched(before, buf, keep, "d2s")


# ---------------------------------------------------------------------------------------------------------------------
# activations through the epilogue: A = 0, so the epilogue sees exactly the bias
# ---------------------------------------------------------------------------------------------------------------------
def _sweep():
    special = [1e-30, 1e-3, 40.0, 1e4, 3e38]
    special = special + [-v for v in special] + [0.0]
    dense = torch.linspace(-10.0, 10.0, 4096 - len(special), dtype=torch.float64)
    return torch.cat([dense, torch.tensor(special, dtype=torch.float64)]).float().cuda()


def _check_act(ops, act, got, x, what):
    x = x.double()
    if act == ops.ACT_RELU:
        _exact(got, x.clamp_min(0), what)
    elif act == ops.ACT_GELU:
        _check_gelu(got, x, what)
    else:  # torch's fp16 recipe
        h = x.half()
        q = (h * torch.sigmoid(1.702 * h)).double()
        nan = torch.isnan(q)
        assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
        g, q = got.double()[~nan], q[~nan]
        fin = torch.isfinite(q)
        assert torch.equal(g[~fin], q[~fin]), f"{what}: infinities differ"
        bad = (g[fin] - q[fin]).abs() > _ulp16(q[fin])
        assert not bad.any(), f"{what}: {int(bad.sum())} values more than 1 fp16 ulp from torch's fp16 QuickGELU"


@pytest.mark.parametrize("act", ["gelu", "quickgelu", "relu"])
def test_activation_sweep(ops, act):
    code = {"gelu": ops.ACT_GELU, "quickgelu": ops.ACT_QUICKGELU, "relu": ops.ACT_RELU}[act]
    v = _sweep()
    N = 128
    M = v.numel() // N
    a = torch.zeros((max(M, 128), 64), dtype=torch.float16, device="cuda")
    wp = ops.pad_rows(_ints((N, 64), -1, 1, 210))
    bias = v.view(M, N)  # one bias row per output row
    o32 = torch.empty((M, N), dtype=torch.float32, device="cuda")
    _plan(ops, {"kernel": K_DIRECT}, "sweep direct", a=a, w=wp, N=N, M=M, bias=bias, bias_group_rows=1, act=code,
          out_f32=o32)
    ops.gemm(a, wp, N, M=M, bias=bias, bias_group_rows=1, act=code, out_f32=o32)
    _check_act(ops, code, o32, bias, f"{act} direct fp32")
    o16 = torch.empty((M, N), dtype=torch.float16, device="cuda")
    _plan(ops, {"kernel": K_TMA_F16}, "sweep tma", a=a, w=wp, N=N, M=M, bias=bias, bias_group_rows=1, act=code,
          out_f16=o16)
    ops.gemm(a, wp, N, M=M, bias=bias, bias_group_rows=1, act=code, out_f16=o16)
    _check_act(ops, code, o16, bias, f"{act} TMA fp16")
    # splitk_reduce_kernel: a zero-input conv on 1 x 1 images, per-column bias, 512 sweep values per call
    Nc, Bc = 512, 4
    x = torch.zeros((Bc, 1, 1, 64), dtype=torch.float16, device="cuda")
    wc = ops.pad_rows(_ints((Nc, 9 * 64), -1, 1, 211))
    for c in range(v.numel() // Nc):
        b = v[c * Nc:(c + 1) * Nc].contiguous()
        r32 = torch.empty((Bc, Nc), dtype=torch.float32, device="cuda")
        r16 = torch.empty((Bc, Nc), dtype=torch.float16, device="cuda")
        kw = dict(conv=(3, 1), bias=b, act=code, out_f32=r32, out_f16=r16)
        if c == 0:
            plan = ops.gemm_plan(x, wc, Nc, **kw)
            if plan["kernel"] != K_FIXED_SPLIT:
                pytest.fail(f"the zero-input conv is not planned as fixed split-K: {plan}")
        ops.gemm(x, wc, Nc, **kw)
        _check_act(ops, code, r32, b.expand(Bc, Nc), f"{act} split-K reduce fp32")
        _check_act(ops, code, r16, b.expand(Bc, Nc), f"{act} split-K reduce fp16")


# ---------------------------------------------------------------------------------------------------------------------
# rejected arguments: an error with a message, and the output untouched
# ---------------------------------------------------------------------------------------------------------------------
def _rejects(ops, match, buf, *args, **kw):
    from lseg_b200._lib import LsegError
    before = buf.clone()
    with pytest.raises(LsegError, match=match):
        ops.gemm(*args, **kw)
    torch.cuda.synchronize()
    _untouched(before, buf, torch.ones_like(buf, dtype=torch.bool), f"rejected call ({match})")


def test_rejected_arguments(ops):
    M, N, K = 256, 128, 64
    a, w = _operands(M, N, K, 220)
    wp = ops.pad_rows(w)
    buf, out = _guarded(M, N, torch.float32)
    a96 = _ints((M, 96), -2, 2, 221)
    _rejects(ops, "multiple of 64", buf, a96, ops.pad_rows(_ints((N, 96), -1, 1, 222)), N, out_f32=out)
    b2, o2 = _guarded(M, 132, torch.float32)
    _rejects(ops, "ldc must be a multiple of 8", b2, a, wp, N, out_f32=o2, ldc=132)
    b16, o16 = _flat(2 * 4 * 4 * 4 * 48, torch.float16)
    _rejects(ops, "depth-to-space", b16, a, ops.pad_rows(_ints((4 * 48, K), -1, 1, 223)), 4 * 48, M=32,
             out_f16=o16, store=ops.STORE_D2S, d2s=(2, 48, 4, 4))
    _rejects(ops, "relu_after_res", buf, a, wp, N, out_f32=out, relu_after_res=True)


@pytest.mark.parametrize("operand", ["bias", "scale", "res_f32", "res2_f32", "res_f16", "out_f32", "out_f16",
                                     "out_f16_relu"])
def test_misaligned_pointer(ops, operand):
    """A contiguous slice such as bias[1:] passes ops.gemm's checks but is not 16-byte aligned: lseg_gemm must refuse it
    by name rather than fault on a vector access."""
    M, N, K = 256, 128, 64
    a, w = _operands(M, N, K, 230)
    wp = ops.pad_rows(w)
    f32 = torch.float32 if operand in ("bias", "scale", "res_f32", "res2_f32", "out_f32") else torch.float16
    base = torch.zeros((M * N + 1,), dtype=f32, device="cuda")
    shifted = base[1:]
    buf, out = _guarded(M, N, torch.float32)
    kw = dict(out_f32=out)
    if operand in ("bias", "scale"):
        kw[operand] = shifted[:N]
    elif operand == "res_f16":
        kw.update(res_f16=shifted.view(M, N), out_f16=torch.zeros((M, N), dtype=torch.float16, device="cuda"))
    elif operand == "out_f32":
        buf = torch.full((M * N + 8,), SENTINEL[torch.float32], dtype=torch.int32, device="cuda").view(torch.float32)
        kw = dict(out_f32=buf[1:M * N + 1].view(M, N))
    else:
        kw[operand] = shifted.view(M, N)
    _rejects(ops, f"{operand} pointer .* not 16-byte aligned", buf, a, wp, N, **kw)
