"""2-CTA clusters of the GEMM (gemm_tc.cuh, CLUSTER): the two CTAs of a pair compute n-tiles 2j and 2j+1 of one m-tile,
and each loads half of the shared A tile into both. Every output element sums the same k16 chunks in the same order as
without clusters, so each case runs one GEMM twice, clustered (lseg_debug_set_gemm_cluster(3): pairs wherever possible,
not only where the planner's rule picks them) and unclustered (mode 1), and requires the two output buffers to be
bit-identical, guard rows included. Operands are random fp16 values, so a wrong A half, a wrong n-tile or a wrong k-chunk
changes bits.

Each case first asserts, through lseg_debug_gemm_cluster, the cluster size its plan runs with (so a build that silently
never clusters cannot pass) and, where it matters, the instantiation (lseg_debug_gemm_plan) and the cluster count. The
planner's own choice (mode 2, the default) is checked on the shapes it was measured on, and the whole forward is compared
across all three modes.
"""
import pytest
import torch

from parity_util import NET_KW, state_dict, synth

pytestmark = pytest.mark.gpu

K_DIRECT, K_TMA_F16, K_TMA_ADD, K_FIXED_SPLIT, K_GROUPED, K_RELU_RES = 0, 1, 2, 3, 4, 5
SENTINEL = {torch.float32: 0x7FC0DEAD, torch.float16: 0x7E5A}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16}
TOKENS = 8 * (30 * 30 + 1)  # ViT-L/16 rows at 480^2, B = 8
NEVER, DEFAULT, ALWAYS = 1, 2, 3  # lseg_debug_set_gemm_cluster modes


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _watchdog(ops):
    yield
    ops.set_gemm_cluster(DEFAULT)
    torch.cuda.synchronize()
    wd = ops.read_watchdog()
    assert wd[0] == 0, f"device barrier watchdog fired: tag={wd[0]} block={wd[1]} thread={wd[2]} parity={wd[3]}"


@pytest.fixture(scope="module")
def pairs(ops):
    """2-CTA clusters the device holds at once (the cluster count of a GEMM with many pair units)."""
    a, w = _rand((128 * 512, 64), 1), ops.pad_rows(_rand((256, 64), 2))
    got = ops.gemm_cluster(a, w, 256, out_f32=torch.empty((128 * 512, 256), device="cuda"))  # K = 64: paired by default
    assert got["cluster"] == 2, got
    return got["clusters"]


def _rand(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _guarded(rows, cols, dtype, fill=None):
    """[rows + 2, cols] of sentinel bits (or a copy of `fill`); returns (buffer, view of rows 1 .. rows)."""
    if fill is None:
        buf = torch.full((rows + 2, cols), SENTINEL[dtype], dtype=BITS[dtype], device="cuda").view(dtype)
    else:
        buf = torch.cat([fill[:1], fill, fill[:1]]).clone()
    return buf, buf[1:rows + 1]


def _flat(n, dtype, guard=64):
    buf = torch.full((n + 2 * guard,), SENTINEL[dtype], dtype=BITS[dtype], device="cuda").view(dtype)
    return buf, buf[guard:guard + n]


def _same(ops, a, w, N, make_out, cluster, kernel=None, clusters=None, **kw):
    """Runs gemm(a, w, N, **kw, **outputs) with pairs wherever possible and unclustered; make_out() -> (dict of output
    keywords, list of guarded buffers). The first plan must have `cluster` (and `kernel`, `clusters` when given); the
    buffers must match."""
    outs, bufs = make_out()
    ops.set_gemm_cluster(ALWAYS)
    try:
        got = ops.gemm_cluster(a, w, N, **kw, **outs)
        assert got["cluster"] == cluster, got
        if clusters is not None:
            assert got["clusters"] == clusters, got
        if kernel is not None:
            plan = ops.gemm_plan(a, w, N, **kw, **outs)
            assert plan["kernel"] == kernel, plan
            assert plan["grid"] == got["clusters"] * got["cluster"], (plan, got)
        ops.gemm(a, w, N, **kw, **outs)
        clustered = [b.clone() for b in bufs]
        outs, bufs = make_out()
        ops.set_gemm_cluster(NEVER)
        assert ops.gemm_cluster(a, w, N, **kw, **outs)["cluster"] == 1
        ops.gemm(a, w, N, **kw, **outs)
    finally:
        ops.set_gemm_cluster(DEFAULT)
    for i, (c, u) in enumerate(zip(clustered, bufs)):
        cb, ub = c.view(BITS[c.dtype]), u.view(BITS[u.dtype])
        n = int((cb != ub).sum())
        assert n == 0, f"output {i}: {n} of {c.numel()} elements differ between the clustered and the unclustered run"
    return clustered


# ---------------------------------------------------------------------------------------------------------------------
# linears: the six instantiations, the ViT-L shapes at B = 8, M tails, small grids, odd unit counts per cluster
# ---------------------------------------------------------------------------------------------------------------------
def _linear(ops, M, N, K, mode, seed, cluster=2, clusters=None, a_rows=None):
    a = _rand((a_rows or M, K), seed)
    w = ops.pad_rows(_rand((N, K), seed + 1, 0.05))
    bias = _rand((N,), seed + 2, 1.0, torch.float32)
    scale = _rand((N,), seed + 3, 0.5, torch.float32).abs() + 0.5
    res = _rand((M, N), seed + 4, 1.0, torch.float32)
    ldc = N
    if mode == "tma_f16":
        kernel, kw = K_TMA_F16, dict(bias=bias, act=ops.ACT_GELU)

        def make():
            b, o = _guarded(M, ldc, torch.float16)
            return dict(out_f16=o), [b]
    elif mode == "tma_add":
        kernel, kw = K_TMA_ADD, dict(bias=bias)

        def make():
            b, x = _guarded(M, ldc, torch.float32, fill=res)
            return dict(res_f32=x, out_f32=x), [b]
    elif mode == "direct":
        kernel, kw = K_DIRECT, dict(bias=bias, scale=scale, res_f32=res)

        def make():
            b32, o32 = _guarded(M, ldc, torch.float32)
            b16, o16 = _guarded(M, ldc, torch.float16)
            return dict(out_f32=o32, out_f16_relu=o16), [b32, b16]
    else:
        assert mode == "relu_res"
        kernel, kw = K_RELU_RES, dict(bias=bias, scale=scale, relu_after_res=True)

        def make():
            b, x = _guarded(M, ldc, torch.float32, fill=res)
            return dict(res_f32=x, out_f32=x), [b]
    _same(ops, a, w, N, make, cluster, kernel=kernel, clusters=clusters, M=M, **kw)


VIT = [(TOKENS, 3072, 1024, "tma_f16"), (TOKENS, 1024, 1024, "tma_add"), (TOKENS, 4096, 1024, "tma_f16"),
       (TOKENS, 1024, 4096, "tma_add")]  # QKV, proj (+= x), fc1 (GELU), fc2 (+= x)


@pytest.mark.parametrize("idx", range(len(VIT)))
def test_vit_linears(ops, idx):
    M, N, K, mode = VIT[idx]
    _linear(ops, M, N, K, mode, 10 + idx)


@pytest.mark.parametrize("mode", ["tma_f16", "tma_add", "direct", "relu_res"])
@pytest.mark.parametrize("M", [1000, 129, 7208 - 64])
def test_linear_m_tails(ops, mode, M):
    """M tails: the last m-tile's A half of rank 1 lies partly (129: wholly) beyond the operand's rows."""
    _linear(ops, M, 512, 192, mode, 20)


def test_linear_a_rows_beyond_m(ops):
    """A has more rows than M: the rows past M reach rank 1's half of the last tile but never the output."""
    _linear(ops, 1000, 256, 128, "direct", 25, a_rows=1100)


def test_fewer_pair_units_than_clusters(ops, pairs):
    """3 m-tiles x 1 n-pair = 3 pair units: 3 clusters, each CTA with one tile (its second warpgroup idle)."""
    assert 3 < pairs
    _linear(ops, 300, 256, 256, "tma_f16", 30, clusters=3)


@pytest.mark.parametrize("extra", [-1, 1])
def test_odd_units_per_cluster(ops, pairs, extra):
    """3 pair units per cluster (warpgroup 0 computes two entries, warpgroup 1 one), one cluster with 2 or 4."""
    m_tiles = 3 * pairs + extra
    _linear(ops, 128 * m_tiles - 5, 256, 320, "direct", 40, clusters=pairs)


@pytest.mark.parametrize("N,mode", [(384, "tma_add"), (128, "tma_f16"), (120, "direct")])
def test_odd_or_single_n_tile_stays_unclustered(ops, N, mode):
    _linear(ops, 2000, N, 256, mode, 50, cluster=1)


@pytest.mark.parametrize("case", ["qkv", "fc2", "one_wave", "one_wave_plus", "odd_n", "head1", "pixel_x_text"])
def test_planner_rule(ops, case):
    """Default mode: pairs when there are more work units than SMs (and the n-tile count is even)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M, K, N, want = {"qkv": (TOKENS, 1024, 3072, 2), "fc2": (TOKENS, 4096, 1024, 2),
                     "one_wave": (128 * (sms // 2), 256, 256, 1),           # units == SMs (even SM count)
                     "one_wave_plus": (128 * (sms // 2) + 1, 256, 256, 2),  # one more m-tile: SMs + 2 units
                     "odd_n": (TOKENS, 512, 384, 1), "head1": (8 * 240 * 240, 256, 512, 2),
                     "pixel_x_text": (8 * 240 * 240, 512, 150, 2)}[case]
    ldc = (N + 7) // 8 * 8
    a, w = _rand((M, K), 55), ops.pad_rows(_rand((N, K), 56))
    got = ops.gemm_cluster(a, w, N, out_f32=torch.empty((M, ldc), device="cuda"), ldc=ldc)
    assert got["cluster"] == want, got


def test_rejected_mode(ops):
    from lseg_b200._lib import LsegError
    for bad in (0, 4, -1):
        with pytest.raises(LsegError, match="mode must be 1, 2 or 3"):
            ops.set_gemm_cluster(bad)


def test_stream_k_stays_unclustered(ops):
    """Stream-K (determinism off) splits K ranges per CTA: never clustered, even with an even n-tile count."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M, N, K = (sms + 5) * 128 - 37, 256, 2112
    a, w = _rand((M, K), 60), ops.pad_rows(_rand((N, K), 61, 0.05))
    x = _rand((M, N), 62, 1.0, torch.float32)
    ops.set_deterministic(False)
    ops.set_gemm_cluster(ALWAYS)
    try:
        plan = ops.gemm_plan(a, w, N, res_f32=x, out_f32=x)
        got = ops.gemm_cluster(a, w, N, res_f32=x, out_f32=x)
    finally:
        ops.set_deterministic(True)
        ops.set_gemm_cluster(DEFAULT)
    assert plan["split_k"] == 1 and got["cluster"] == 1, (plan, got)


# ---------------------------------------------------------------------------------------------------------------------
# implicit-GEMM 3x3 convs at the decoder levels (B = 8); 15^2 runs the fixed split-K schedule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side", [120, 60, 30, 15])
@pytest.mark.parametrize("kind", ["conv_f16", "conv_direct"])
def test_conv3x3(ops, side, kind):
    B, C, N = 8, 256, 256
    P = B * side * side
    x = _rand((B, side, side, C), 70 + side)
    w = ops.pad_rows(_rand((N, 9 * C), 71, 0.02))
    sc = _rand((N,), 72, 0.5, torch.float32).abs() + 0.5
    sh = _rand((N,), 73, 1.0, torch.float32)
    res = _rand((P, N), 74, 1.0, torch.float32)
    if kind == "conv_f16":
        kw = dict(conv=(3, 1), scale=sc, bias=sh, act=ops.ACT_RELU, ldc=N)

        def make():
            b, o = _guarded(P, N, torch.float16)
            return dict(out_f16=o), [b]
    else:
        kw = dict(conv=(3, 1), scale=sc, bias=sh, res_f32=res, ldc=N)

        def make():
            b32, o32 = _guarded(P, N, torch.float32)
            b16, o16 = _guarded(P, N, torch.float16)
            return dict(out_f32=o32, out_f16_relu=o16), [b32, b16]
    outs, _ = make()
    plan = ops.gemm_plan(x, w, N, **kw, **outs)
    if side == 15:
        assert plan["kernel"] == K_FIXED_SPLIT, plan
    _same(ops, x, w, N, make, 2, **kw)


def test_conv3x3_wide_input(ops):
    """layer4_rn-like: 15^2, 1024 input channels (144 k-chunks) on the fixed split-K schedule; H = 15 puts pixel row 15
    of every second m-tile (rank 1's half) outside the image."""
    B, C, N = 8, 1024, 256
    x = _rand((B, 15, 15, C), 80)
    w = ops.pad_rows(_rand((N, 9 * C), 81, 0.02))

    def make():
        b32, o32 = _guarded(B * 225, N, torch.float32)
        b16, o16 = _guarded(B * 225, N, torch.float16)
        return dict(out_f32=o32, out_f16_relu=o16), [b32, b16]
    _same(ops, x, w, N, make, 2, kernel=K_FIXED_SPLIT, conv=(3, 1), ldc=N)


# ---------------------------------------------------------------------------------------------------------------------
# stores: pixel x text (NCHW, N = 150 = a full tile and a 22-column one), grouped NCHW, depth-to-space
# ---------------------------------------------------------------------------------------------------------------------
def test_pixel_x_text(ops):
    B, P, D, K = 8, 240 * 240, 512, 150
    feat = _rand((B * P, D), 90)
    text = ops.pad_rows(_rand((K, D), 91, 0.05))
    ss = (torch.rand((B * P, D // 32), generator=torch.Generator().manual_seed(92)) + 0.5).cuda()

    def make():
        b, o = _flat(B * K * P, torch.float16)
        return dict(out_f16=o.view(B, K, P)), [b]
    _same(ops, feat, text, K, make, 2, kernel=K_DIRECT, store=ops.STORE_NCHW_T, nchw=(P, K), row_sumsq=ss,
          row_scale=14.0)


def test_grouped_nchw(ops):
    B, P, D, stride, K = 8, 900, 512, 32, 30  # N = 256: two n-tiles, image blocks of 32 columns
    a = _rand((B * P, D), 95)
    w = ops.pad_rows(_rand((B * stride, D), 96, 0.05))

    def make():
        b, o = _flat(B * K * P, torch.float16)
        return dict(out_f16=o.view(B, K, P)), [b]
    _same(ops, a, w, B * stride, make, 2, kernel=K_GROUPED, store=ops.STORE_NCHW_T, nchw=(P, K, stride))


@pytest.mark.parametrize("s,cout,g", [(4, 256, 30), (2, 512, 60), (8, 128, 15)])
def test_depth_to_space(ops, s, cout, g):
    B, cin = 8, 1024
    N = s * s * cout
    a = _rand((B * g * g, cin), 100 + s)
    w = ops.pad_rows(_rand((N, cin), 101, 0.05))
    bias = _rand((cout,), 102, 1.0, torch.float32).repeat(s * s).contiguous()

    def make():
        b, o = _flat(B * (g * s) ** 2 * cout, torch.float16)
        return dict(out_f16=o), [b]
    _same(ops, a, w, N, make, 2, kernel=K_DIRECT, bias=bias, store=ops.STORE_D2S, d2s=(s, cout, g, g), M=B * g * g)


# ---------------------------------------------------------------------------------------------------------------------
# the whole forward at the benchmark's size
# ---------------------------------------------------------------------------------------------------------------------
def test_forward_480_k150(ops):
    from lseg_b200.lseg_net import LSegNet
    net = LSegNet(labels=synth.ade20k_labels(), **NET_KW)
    net.load_state_dict(state_dict(0))
    net = net.cuda().eval()
    tokens = synth.tokenize(synth.ade20k_labels())
    assert len(synth.ade20k_labels()) == 150
    x = synth.make_image(8, 480, 480, seed=7).cuda()
    out = {}
    try:
        for mode in (DEFAULT, NEVER, ALWAYS):
            ops.set_gemm_cluster(mode)
            out[mode] = net(x, tokens)
    finally:
        ops.set_gemm_cluster(DEFAULT)
    assert out[NEVER].dtype == torch.float32
    for mode in (DEFAULT, ALWAYS):
        assert torch.equal(out[mode].view(torch.int32), out[NEVER].view(torch.int32)), \
            f"mode {mode}: max |diff| {(out[mode] - out[NEVER]).abs().max().item()}"
