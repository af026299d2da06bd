"""The TMA epilogues (fp16 store, fp32 reduce-add) against the register-direct epilogue, bit for bit.

Both epilogues apply the same arithmetic to the same accumulators: the K loop, and with it every accumulator bit, does
not depend on the epilogue. The TMA epilogues take each warp's wgmma fragment straight into 16-row TMA boxes, so a wrong
fragment row / column, swizzle or box coordinate shows up as a bit difference against the register-direct path, which
stages the accumulators and maps threads to rows. An extra output forces a GEMM onto the register-direct path: out_f32
beside out_f16, or an fp32 residual that is not the output (acc * s + b + x there, x + (acc * s + b) through the
reduce-add: the same fp32 sum). Operands are random fp16 values, so every rounding point matters; the stream-K cases use
small integers instead, because a split tile sums its k-segments in another order (exact for integers).

GEMMs with row sums (out_row_sumsq, head1) keep the fp16 TMA store but stage their accumulators first, so that a thread
holds whole rows and sums them in column order; those cases check that form against the register-direct path.

Every output sits between two 4 KiB guard bands of sentinel bits, and the padding columns past N must keep their bits.
Every case asserts the plan it is meant to exercise.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_DIRECT, EPI_TMA_F16, EPI_TMA_ADD = 0, 1, 2
K_DIRECT, K_TMA_F16, K_TMA_ADD = 0, 1, 2
SENTINEL = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7E5A}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16}
GUARD_BYTES = 4096


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
def cluster_mode(ops, request):
    ops.set_gemm_cluster(request.param)
    try:
        yield request.param
    finally:
        ops.set_gemm_cluster(2)


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _randh(shape, seed, s=0.5):
    return (torch.randn(shape, generator=_gen(seed)) * s).half().cuda()


def _randf(shape, seed):
    return torch.randn(shape, generator=_gen(seed)).cuda()


def _ints(shape, lo, hi, seed, dtype=torch.float16):
    return torch.randint(lo, hi + 1, shape, generator=_gen(seed)).to(dtype).cuda()


class Guarded:
    """rows x ldc output inside a flat buffer with GUARD_BYTES of sentinel bits (or a copy of `fill`) on each side."""

    def __init__(self, rows, ldc, dtype, fill=None):
        self.g = GUARD_BYTES // torch.tensor([], dtype=dtype).element_size()
        self.n = rows * ldc
        self.buf = torch.full((self.n + 2 * self.g,), SENTINEL[dtype], dtype=BITS[dtype], device="cuda").view(dtype)
        self.out = self.buf[self.g:self.g + self.n].view(rows, ldc)
        if fill is not None:
            self.out.copy_(fill)
        self.before = self.buf.clone()

    def check_outside(self, N, what):
        keep = torch.ones_like(self.buf, dtype=torch.bool)
        keep[self.g:self.g + self.n].view(self.out.shape)[:, :N] = False
        b, a = self.before.view(BITS[self.buf.dtype]), self.buf.view(BITS[self.buf.dtype])
        bad = int(((a != b) & keep).sum())
        assert bad == 0, f"{what}: {bad} elements outside the output window were written"


def _same_bits(got, want, what):
    g, w = got.contiguous().view(BITS[got.dtype]), want.contiguous().view(BITS[want.dtype])
    bad = g != w
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {n} of {got.numel()} elements differ; first at {idx}: "
                             f"got {got[tuple(idx)].item()}, want {want[tuple(idx)].item()}")


def _plan(ops, want, what, a, w, N, **kw):
    got = ops.gemm_plan(a, w, N, **kw)
    for k, v in want.items():
        assert got[k] == v, f"{what}: plan {got}, expected {k} = {v}"
    return got


def _f16_vs_direct(ops, a, wp, N, rows, ldc, what, sumsq=False, **kw):
    """The fp16 TMA store against the register-direct store of the same GEMM (+ the row sums of squares)."""
    parts = (N + 31) // 32
    t16 = Guarded(rows, ldc, torch.float16)
    d16, d32 = Guarded(rows, ldc, torch.float16), Guarded(rows, ldc, torch.float32)
    tss = Guarded(rows, parts, torch.float32) if sumsq else None
    dss = Guarded(rows, parts, torch.float32) if sumsq else None
    tkw = dict(kw, out_f16=t16.out, ldc=ldc)
    dkw = dict(kw, out_f16=d16.out, out_f32=d32.out, ldc=ldc)
    if sumsq:
        tkw["out_row_sumsq"], dkw["out_row_sumsq"] = tss.out, dss.out
    _plan(ops, {"kernel": K_TMA_F16, "epi": EPI_TMA_F16, "split_fixed": 0}, what, a, wp, N, **tkw)
    _plan(ops, {"kernel": K_DIRECT, "epi": EPI_DIRECT, "split_fixed": 0}, what + " (reference)", a, wp, N, **dkw)
    ops.gemm(a, wp, N, **tkw)
    ops.gemm(a, wp, N, **dkw)
    torch.cuda.synchronize()
    assert not torch.isnan(d16.out[:, :N]).any(), f"{what}: reference left sentinels"
    _same_bits(t16.out[:, :N], d16.out[:, :N], what)
    t16.check_outside(N, what)
    if sumsq:
        _same_bits(tss.out, dss.out, what + " row sumsq")
        tss.check_outside(parts, what + " row sumsq")


def _add_vs_direct(ops, a, wp, N, M, ldc, x0, what, plan_want=None, **kw):
    """The in-place fp32 reduce-add (x += epi(A W^T)) against the register-direct store of x + epi(A W^T)."""
    t = Guarded(M, ldc, torch.float32, fill=x0)
    d = Guarded(M, ldc, torch.float32)
    want = {"kernel": K_TMA_ADD, "epi": EPI_TMA_ADD, "split_k": 0}
    want.update(plan_want or {})
    _plan(ops, want, what, a, wp, N, M=M, res_f32=t.out, out_f32=t.out, ldc=ldc, **kw)
    _plan(ops, {"kernel": K_DIRECT, "epi": EPI_DIRECT}, what + " (reference)", a, wp, N, M=M, res_f32=x0, out_f32=d.out,
          ldc=ldc, **kw)
    ops.gemm(a, wp, N, M=M, res_f32=t.out, out_f32=t.out, ldc=ldc, **kw)
    ops.gemm(a, wp, N, M=M, res_f32=x0, out_f32=d.out, ldc=ldc, **kw)
    torch.cuda.synchronize()
    _same_bits(t.out[:, :N], d.out[:, :N], what)
    t.check_outside(N, what)


M_TAILS = [1, 15, 16, 17, 63, 64, 65, 127]
N_LIST = [64, 136, 200, 1024, 3072]


def _act(ops, i):
    return (ops.ACT_NONE, ops.ACT_GELU, ops.ACT_QUICKGELU, ops.ACT_RELU)[i % 4]


@pytest.mark.parametrize("N", N_LIST)
@pytest.mark.parametrize("tail", M_TAILS)
def test_f16_tails(ops, tail, N):
    M, K = 2 * 128 + tail, 192
    i = M_TAILS.index(tail) + N_LIST.index(N)
    a, wp = _randh((M + 40, K), 1 + i), ops.pad_rows(_randh((N, K), 2 + i, 0.1))
    kw = dict(M=M, bias=_randf((N,), 3 + i), act=_act(ops, i))
    if i % 2:
        kw["scale"] = _randf((N,), 4 + i)
    _f16_vs_direct(ops, a, wp, N, M, N + 8, f"f16 M={M} N={N}", sumsq=(tail in (1, 17, 65)), **kw)


@pytest.mark.parametrize("N", N_LIST)
@pytest.mark.parametrize("tail", M_TAILS)
def test_add_tails(ops, tail, N):
    M, K, ldc = 2 * 128 + tail, 256, N + 8
    i = M_TAILS.index(tail) + N_LIST.index(N)
    a, wp = _randh((M, K), 11 + i), ops.pad_rows(_randh((N, K), 12 + i, 0.1))
    x0 = _randf((M, ldc), 13 + i)
    kw = dict(bias=_randf((N,), 14 + i), act=_act(ops, i))
    if i % 2:
        kw["scale"] = _randf((N,), 15 + i)
    _add_vs_direct(ops, a, wp, N, M, ldc, x0, f"add M={M} N={N}", **kw)


@pytest.mark.parametrize("act", ["none", "gelu", "quickgelu", "relu"])
@pytest.mark.parametrize("mode", ["f16", "add"])
def test_activations(ops, mode, act):
    M, N, K = 1000, 512, 1024
    code = {"none": ops.ACT_NONE, "gelu": ops.ACT_GELU, "quickgelu": ops.ACT_QUICKGELU, "relu": ops.ACT_RELU}[act]
    a, wp = _randh((M, K), 21), ops.pad_rows(_randh((N, K), 22, 0.05))
    kw = dict(bias=_randf((N,), 23), scale=_randf((N,), 24), act=code)
    if mode == "f16":
        _f16_vs_direct(ops, a, wp, N, M, N, f"f16 {act}", M=M, **kw)
    else:
        _add_vs_direct(ops, a, wp, N, M, N, _randf((M, N), 25), f"add {act}", **kw)


@pytest.mark.parametrize("N", [64, 136, 200, 512])
def test_row_sumsq_order(ops, N):
    """head1's partial squared row norms: each 32-column chunk summed in column order, bit for bit."""
    M, K = 3000, 256
    a, wp = _randh((M, K), 31), ops.pad_rows(_randh((N, K), 32, 0.1))
    _f16_vs_direct(ops, a, wp, N, M, N, f"sumsq N={N}", sumsq=True, M=M, bias=_randf((N,), 33))


@pytest.mark.parametrize("group_rows,B", [(900, 3), (225, 8), (100, 5)])
@pytest.mark.parametrize("mode", ["f16", "add"])
def test_grouped_bias(ops, mode, group_rows, B):
    """Per-image bias rows whose groups straddle tiles (and, at 100 rows, the 16-row fragment blocks)."""
    M, N, K = group_rows * B, 1024, 192
    a, wp = _randh((M, K), 41), ops.pad_rows(_randh((N, K), 42, 0.1))
    kw = dict(bias=_randf((B, N), 43), bias_group_rows=group_rows, act=ops.ACT_GELU)
    if mode == "f16":
        _f16_vs_direct(ops, a, wp, N, M, N, f"grouped f16 G={group_rows}", M=M, **kw)
    else:
        _add_vs_direct(ops, a, wp, N, M, N, _randf((M, N), 44), f"grouped add G={group_rows}", **kw)


CONVS = [  # B, H, W, Cin, N, (ksize, pad): no split-K at these shapes (gemm_pick_split)
    (2, 15, 15, 256, 256, (1, 0)), (2, 30, 30, 256, 128, (1, 0)), (2, 60, 60, 64, 256, (3, 1)),
    (1, 120, 120, 64, 128, (3, 1)), (2, 17, 33, 64, 192, (3, 1)), (3, 13, 21, 128, 72, (1, 0))]


@pytest.mark.parametrize("idx", range(len(CONVS)))
def test_conv(ops, idx):
    B, H, W, Cin, N, conv = CONVS[idx]
    x = _randh((B, H, W, Cin), 51 + idx)
    wp = ops.pad_rows(_randh((N, conv[0] * conv[0] * Cin), 52 + idx, 0.05))
    kw = dict(conv=conv, scale=_randf((N,), 53 + idx), bias=_randf((N,), 54 + idx), act=_act(ops, idx))
    _f16_vs_direct(ops, x, wp, N, B * H * W, N + 16, f"conv {B}x{H}x{W}x{Cin} -> {N} k{conv[0]}", **kw)


@pytest.mark.parametrize("cluster_mode", [1, 3], indirect=True)
def test_cluster_modes(ops, cluster_mode):
    """Unclustered and 2-CTA-cluster plans of the same GEMMs."""
    M, N, K = 2000 + 37, 1024, 512
    a, wp = _randh((M, K), 61), ops.pad_rows(_randh((N, K), 62, 0.05))
    bias = _randf((N,), 63)
    want = 2 if cluster_mode == 3 else 1
    o16, x = torch.empty(M, N, dtype=torch.float16, device="cuda"), torch.zeros(M, N, device="cuda")
    for what, kw in (("f16", dict(out_f16=o16)), ("add", dict(res_f32=x, out_f32=x))):
        got = ops.gemm_cluster(a, wp, N, M=M, bias=bias, **kw)
        assert got["cluster"] == want, f"{what}: {got}"
    _f16_vs_direct(ops, a, wp, N, M, N, f"f16 cluster mode {cluster_mode}", M=M, bias=bias, act=ops.ACT_GELU)
    _add_vs_direct(ops, a, wp, N, M, N, _randf((M, N), 64), f"add cluster mode {cluster_mode}", bias=bias)
    x = _randh((2, 60, 60, 64), 65)
    wc = ops.pad_rows(_randh((256, 9 * 64), 66, 0.05))
    kw = dict(conv=(3, 1), scale=_randf((256,), 67), bias=_randf((256,), 68), act=ops.ACT_RELU)
    got = ops.gemm_cluster(x, wc, 256, out_f16=torch.empty(7200, 256, dtype=torch.float16, device="cuda"), **kw)
    assert got["cluster"] == want, f"conv: {got}"
    _f16_vs_direct(ops, x, wc, 256, 7200, 256, f"conv cluster mode {cluster_mode}", **kw)


@pytest.mark.parametrize("k_iters", [32, 33, 35])
def test_stream_k(ops, sms, k_iters):
    """Stream-K reduce-add (determinism off): tiles split across CTAs, the bias added by the k = 0 segment only."""
    M, N, ldc = (sms + 5) * 128 - 37, 128, 136
    K = 64 * k_iters
    a, wp = _ints((M, K), -2, 2, 71 + k_iters), ops.pad_rows(_ints((N, K), -1, 1, 72 + k_iters))
    x0 = (_ints((M, ldc), -32, 32, 73, torch.float32) * 0.25)
    bias = _ints((N,), -32, 32, 74, torch.float32) * 0.25
    ops.set_deterministic(False)
    try:
        _add_vs_direct(ops, a, wp, N, M, ldc, x0, f"stream-K k_iters={k_iters}", plan_want={"split_k": 1}, bias=bias)
    finally:
        ops.set_deterministic(True)
