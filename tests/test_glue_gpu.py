"""The glue kernels of the forward path, element by element, at the shapes where they can go wrong.

Every output is written into a view of a larger byte buffer filled with a sentinel pattern (0xA5 bytes), 4 KiB past
its start and 4 KiB before its end, so a store outside the output, or into padding the caller relies on, is seen. Data-movement kernels are
compared bit for bit; the arithmetic ones against the float64 references and bounds of tests/glue_oracle.py. Variants
that promise the same values (smem line layouts, streaming stores, the shared-memory-free upsample) must give the same
bits, two runs the same bits, and changing one image of a batch must leave the others' outputs untouched.
"""
import ctypes as C
import math
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as F

import glue_oracle as G

pytestmark = pytest.mark.gpu

SENT = 0xA5
# bytes of guard band before and after every output: wider than the widest store unit (one 1 KiB fp32 pixel of the
# C = 256 decoder kernels), so a store one pixel or row-tail past the output lands in the band, not in another tensor;
# a multiple of 16 keeps the output's alignment
PAD = 4096
LS = math.exp(math.log(1 / 0.07))


@pytest.fixture(scope="module")
def ops():
    import lseg_b200  # noqa: F401
    from lseg_b200 import ops as _ops
    return _ops


class Guarded:
    """A contiguous `dtype` tensor of `shape` inside a sentinel-filled byte buffer with PAD bytes on either side."""

    def __init__(self, shape, dtype):
        self.n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        self.buf = torch.full((self.n + 2 * PAD,), SENT, dtype=torch.uint8, device="cuda")
        self.t = self.buf[PAD:PAD + self.n].view(dtype).view(shape)

    def check(self, what):
        torch.cuda.synchronize()
        lo, hi = self.buf[:PAD], self.buf[PAD + self.n:]
        assert bool((lo == SENT).all()) and bool((hi == SENT).all()), f"{what}: a store landed in the guard band"


def _rand(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _bound_ok(got, ref, bound, what):
    n, msg = G.violations(got, ref, bound)
    assert n == 0, f"{what}: {msg}"


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                     b.contiguous().view(torch.uint8))


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm
# ---------------------------------------------------------------------------------------------------------------
def _ln_input(M, C, dtype, seed):
    x = _rand((M, C), seed, 2.0) + 0.5
    if M > 1:
        x[1] = 300.0 + _rand((C,), seed + 1, 0.05)  # |mean| >> std
    if M > 2:
        x[2] = 7.0  # constant row: variance 0, eps alone
    if M > 3:
        x[3] = 0.5 + _rand((C,), seed + 2, 1e-3)  # variance near eps
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [512, 768, 1024])
@pytest.mark.parametrize("M", [1, 7, 8, 9])
def test_layernorm_block_edges(ops, M, C, dtype):
    x = _ln_input(M, C, dtype, M * 7 + C)
    g, b = _rand((C,), 1), _rand((C,), 2, 0.1)
    eps = 1e-6 if dtype == torch.float32 else 1e-5
    y = Guarded((M, C), torch.float16)
    ops.layernorm(x, g, b, eps, out=y.t)
    y.check("layernorm")
    _bound_ok(y.t, *G.layernorm_ref(x, g, b, eps), f"layernorm M={M} C={C} {dtype}")


@pytest.mark.parametrize("M,C,dtype", [(7208, 1024, torch.float32), (8 * 226, 768, torch.float32),
                                       (150 * 77, 512, torch.float16)])
def test_layernorm_engine_shapes(ops, M, C, dtype):
    x = _ln_input(M, C, dtype, 5)
    g, b = _rand((C,), 3), _rand((C,), 4, 0.1)
    eps = 1e-6 if dtype == torch.float32 else 1e-5
    y = Guarded((M, C), torch.float16)
    ops.layernorm(x, g, b, eps, out=y.t)
    y.check("layernorm")
    _bound_ok(y.t, *G.layernorm_ref(x, g, b, eps), f"layernorm M={M} C={C}")
    assert _bits_equal(ops.layernorm(x, g, b, eps), y.t), "layernorm: two runs differ"


# ---------------------------------------------------------------------------------------------------------------
# ViT glue: patchify, pos_resize, assemble_tokens, readout_split
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,P", [(8, 480, 480, 16), (1, 736, 736, 16), (2, 480, 480, 32), (2, 64, 96, 16),
                                     (1, 32, 32, 32)])
def test_patchify_exact(ops, B, H, W, P):
    x = _rand((B, 3, H, W), 10)
    a = Guarded((B * (H // P) * (W // P), 3 * P * P), torch.float16)
    ops.patchify(x, P, out=a.t)
    a.check("patchify")
    ref = F.unfold(x, P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P).half()
    assert _bits_equal(a.t, ref), f"patchify P={P}"


@pytest.mark.parametrize("g0,gh,gw,D", [(24, 30, 30, 1024), (24, 46, 46, 1024), (24, 4, 6, 1024), (24, 15, 23, 1024),
                                        (12, 15, 15, 768), (12, 6, 9, 768), (12, 1, 1, 768)])
def test_pos_resize(ops, g0, gh, gw, D):
    pos = _rand((1 + g0 * g0, D), 11, 0.02)
    out = Guarded((1 + gh * gw, D), torch.float32)
    ops.pos_resize(pos, g0, gh, gw, out=out.t)
    out.check("pos_resize")
    assert _bits_equal(out.t[0], pos[0]), "pos_resize cls row"
    grid = pos[1:].view(g0, g0, D).permute(2, 0, 1)
    ref, absum, slack = G.bilinear_ref(grid, gh, gw, False, contract_slack=True)
    ref, bound = G.bilinear_bound(ref, absum, slack)
    _bound_ok(out.t[1:].view(gh, gw, D).permute(2, 0, 1), ref, bound, f"pos_resize {g0}->{gh}x{gw}")


@pytest.mark.parametrize("B,T,D", [(8, 900, 1024), (2, 225, 768), (3, 5, 4)])
def test_assemble_readout_exact(ops, B, T, D):
    patch, cls, pos = _rand((B * T, D), 12), _rand((D,), 13), _rand((T + 1, D), 14, 0.02)
    x = Guarded((B, T + 1, D), torch.float32)
    ops.assemble_tokens(patch, cls, pos, B, T, out=x.t)
    x.check("assemble_tokens")
    ref = torch.cat([cls.view(1, 1, D).expand(B, 1, D), patch.view(B, T, D)], 1) + pos
    assert _bits_equal(x.t, ref), "assemble_tokens"
    rows = (B + 127) // 128 * 128
    tok, cl = Guarded((B * T, D), torch.float16), Guarded((rows, D), torch.float16)
    ops.readout_split(x.t, out=(tok.t, cl.t))
    tok.check("readout_split tok")
    cl.check("readout_split cls")
    assert _bits_equal(tok.t, ref[:, 1:].reshape(B * T, D).half()), "readout_split tok"
    assert _bits_equal(cl.t[:B], ref[:, 0].half()), "readout_split cls"
    assert bool((cl.t[B:].view(torch.uint8) == SENT).all()), "readout_split wrote into the cls padding rows"


# ---------------------------------------------------------------------------------------------------------------
# NHWC data movement: im2col_3x3_s2, stem_im2col, maxpool, subsample
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C", [(8, 60, 60, 256), (2, 30, 30, 256), (1, 7, 5, 8), (3, 1, 1, 64), (1, 4, 9, 264)])
def test_im2col_3x3_s2_exact(ops, B, H, W, C):
    x = _rand((B, H, W, C), 15, dtype=torch.float16)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    a = Guarded((B * Ho * Wo, 9 * C), torch.float16)
    ops.im2col_3x3_s2(x, out=a.t)
    a.check("im2col_3x3_s2")
    cols = F.unfold(x.float().permute(0, 3, 1, 2), 3, padding=1, stride=2)  # [B, C*9, L], row c*9 + tap
    ref = cols.view(B, C, 9, Ho * Wo).permute(0, 3, 2, 1).reshape(B * Ho * Wo, 9 * C).half()
    assert _bits_equal(a.t, ref), "im2col_3x3_s2 (tap-major columns)"


@pytest.mark.parametrize("B,H,W", [(2, 480, 480), (1, 64, 96), (1, 2, 2), (3, 6, 10)])
def test_stem_im2col_exact(ops, B, H, W):
    x = _rand((B, 3, H, W), 16)
    a = Guarded((B * (H // 2) * (W // 2), 192), torch.float16)
    ops.stem_im2col(x, out=a.t)
    a.check("stem_im2col")
    ref = F.unfold(x, 7, padding=3, stride=2).transpose(1, 2).reshape(-1, 147).half()
    assert _bits_equal(a.t[:, :147].contiguous(), ref), "stem_im2col columns 0..146"
    assert bool((a.t[:, 147:].view(torch.int16) == 0).all()), "stem_im2col zero columns 147..191"


@pytest.mark.parametrize("B,H,W,C,neg", [(2, 240, 240, 64, False), (1, 2, 2, 8, True), (3, 6, 10, 264, True),
                                         (1, 120, 184, 256, False)])
def test_maxpool_subsample_exact(ops, B, H, W, C, neg):
    x = _rand((B, H, W, C), 17, dtype=torch.float16)
    if neg:  # all values negative: a zero-padded window would win at every border
        x = -x.abs() - 1
    y = Guarded((B, H // 2, W // 2, C), torch.float16)
    ops.maxpool3x3s2_nhwc(x, out=y.t)
    y.check("maxpool3x3s2_nhwc")
    ref = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).half()
    assert _bits_equal(y.t, ref), "maxpool3x3s2_nhwc"
    s = Guarded((B, H // 2, W // 2, C), torch.float16)
    ops.subsample2_nhwc(x, out=s.t)
    s.check("subsample2_nhwc")
    assert _bits_equal(s.t, x[:, ::2, ::2].contiguous()), "subsample2_nhwc"


# ---------------------------------------------------------------------------------------------------------------
# NHWC bilinear x2: the generic kernel and the C = 256 decoder kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [8, 64, 264])
@pytest.mark.parametrize("H,W", [(1, 1), (2, 3), (3, 15), (2, 16), (1, 17), (15, 15)])
def test_upsample2x_nhwc_generic(ops, H, W, C):
    x = _rand((2, H, W, C), 18, 2.0, torch.float16)
    y = Guarded((2, 2 * H, 2 * W, C), torch.float16)
    ops.upsample2x_nhwc(x, out=y.t)
    y.check("upsample2x_nhwc")
    ref, bound = G.upsample2x_ref(x.permute(0, 3, 1, 2), out_f16=True)
    _bound_ok(y.t.permute(0, 3, 1, 2), ref, bound, f"upsample2x_nhwc {H}x{W}x{C}")


# output variants of the C = 256 decoder kernels: fp32, fp16, and fp32 with the fp32 skip operand summed in
NHWC256_OUTS = {"f32": (torch.float32, False), "f16": (torch.float16, False), "f32_add": (torch.float32, True)}


def _nhwc256_case(ops, x, out, what):
    """One output variant against the oracle; returns the result."""
    B, H, W, _ = x.shape
    out_dtype, with_add = NHWC256_OUTS[out]
    skip = _rand((B, 2 * H, 2 * W, 256), 19) if with_add else None
    y = Guarded((B, 2 * H, 2 * W, 256), out_dtype)
    ops.upsample2x_nhwc(x, out_dtype, add=skip, decoder=True, out=y.t)
    y.check(what)
    ref, bound = G.upsample2x_ref(x.permute(0, 3, 1, 2), add=None if skip is None else skip.permute(0, 3, 1, 2),
                                  out_f16=out_dtype == torch.float16)
    _bound_ok(y.t.permute(0, 3, 1, 2), ref, bound, f"{what} out {out}")
    return y.t


@pytest.mark.parametrize("out", list(NHWC256_OUTS))
@pytest.mark.parametrize("src", [torch.float16, torch.float32])
@pytest.mark.parametrize("H", [1, 2, 3])
@pytest.mark.parametrize("W", [1, 2, 3, 15, 16, 17, 31, 33])
def test_upsample2x_nhwc256_block_edges(ops, W, H, src, out):
    """2W ends at every position of the 4-pixel warp group and of the 32-pixel block."""
    _nhwc256_case(ops, _rand((2, H, W, 256), 20, 2.0, src), out, f"upsample2x_nhwc256 {H}x{W} {src}")


@pytest.mark.parametrize("out", list(NHWC256_OUTS))
@pytest.mark.parametrize("B,h", [(2, 15), (2, 30), (1, 60), (1, 120), (1, 23), (1, 46), (1, 92), (1, 184)])
def test_upsample2x_nhwc256_decoder_levels(ops, B, h, out):
    x = _rand((B, h, h, 256), 21, 2.0, torch.float16)
    got = _nhwc256_case(ops, x, out, f"upsample2x_nhwc256 level {h}")
    if B > 1 and out == "f32":  # image independence
        x2 = x.clone()
        x2[0] = -x2[0]
        again = ops.upsample2x_nhwc(x2, torch.float32, decoder=True)
        assert _bits_equal(again[1:], got[1:]), "upsample2x_nhwc256: image 1 changed with image 0"


# ---------------------------------------------------------------------------------------------------------------
# NCHW logits upsample and its variants
# ---------------------------------------------------------------------------------------------------------------
NCHW_SHAPES = [(1, 3, 1, 8), (2, 2, 2, 16), (1, 2, 17, 504), (1, 2, 17, 512), (1, 3, 2, 512), (2, 5, 120, 120),
               (1, 4, 184, 184), (1, 65535, 1, 8)]


@pytest.mark.parametrize("B,K,H,W", NCHW_SHAPES)
def test_upsample2x_nchw(ops, B, K, H, W):
    x = _rand((B, K, H, W), 22, 3.0, torch.float16)
    y = Guarded((B, K, 2 * H, 2 * W), torch.float32)
    ops.upsample2x_nchw(x, out=y.t)
    y.check("upsample2x_nchw")
    _bound_ok(y.t, *G.upsample2x_ref(x), f"upsample2x_nchw {B}x{K}x{H}x{W}")
    from lseg_b200 import _lib
    lib = _lib.load()
    old = lib.lseg_debug_upsample_layout(1)
    try:
        split = ops.upsample2x_nchw(x)
    finally:
        lib.lseg_debug_upsample_layout(old)
    assert _bits_equal(split, y.t), "upsample2x_nchw: split and interleaved smem layouts differ"
    bg = Guarded((B, K, 2 * H, 2 * W), torch.float32)
    ops.upsample2x_nchw(x, background=True, out=bg.t)
    bg.check("upsample2x_nchw_bg")
    assert _bits_equal(bg.t, y.t), "upsample2x_nchw and upsample2x_nchw_bg differ"
    f = x.float()
    y32 = Guarded((B, K, 2 * H, 2 * W), torch.float32)
    ops.upsample2x_nchw_f32(f, out=y32.t)
    y32.check("upsample2x_nchw_f32")
    assert _bits_equal(y32.t, y.t), "fp32-input upsample differs on fp16-representable values"
    assert _bits_equal(ops.upsample2x_nchw(x), y.t), "upsample2x_nchw: two runs differ"
    if B > 1:
        x2 = x.clone()
        x2[0] = 0
        assert _bits_equal(ops.upsample2x_nchw(x2)[1:], y.t[1:]), "upsample2x_nchw: image 1 changed with image 0"


@pytest.mark.parametrize("B,K,H,W", [(1, 3, 17, 512), (2, 5, 23, 8), (1, 4, 120, 120)])
def test_upsample2x_nchw_f32_bound(ops, B, K, H, W):
    x = _rand((B, K, H, W), 23, 3.0)
    y = Guarded((B, K, 2 * H, 2 * W), torch.float32)
    ops.upsample2x_nchw_f32(x, out=y.t)
    y.check("upsample2x_nchw_f32")
    _bound_ok(y.t, *G.upsample2x_ref(x), "upsample2x_nchw_f32")


_CS_SCRIPT = """
import sys, torch
sys.path.insert(0, sys.argv[1])
import lseg_b200
from lseg_b200 import ops
x = torch.load(sys.argv[2])
torch.save(ops.upsample2x_nchw(x.cuda()).cpu(), sys.argv[3])
"""


def test_upsample2x_nchw_streaming_stores_same_bits(ops):
    """LSEG_UPSAMPLE_CS=1 selects the st.global.cs instantiation once per process: a subprocess runs it."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    x = _rand((2, 3, 17, 512), 24, 3.0, torch.float16)
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "x.pt"), os.path.join(d, "y.pt")
        torch.save(x.cpu(), src)
        env = dict(os.environ, LSEG_UPSAMPLE_CS="1")
        subprocess.run([sys.executable, "-c", _CS_SCRIPT, root, src, dst], env=env, check=True, timeout=600)
        cs = torch.load(dst)
    assert _bits_equal(cs, ops.upsample2x_nchw(x).cpu()), "streaming-store instantiation differs"


@pytest.mark.parametrize("B,K,H,W", [(2, 5, 2, 512), (1, 3, 17, 504), (2, 4, 1, 8), (1, 150, 30, 16)])
def test_upsample2x_argmax_block_edges(ops, B, K, H, W):
    x = ((_rand((B, K, H, W), 25, 2.0) * 4).round() / 4).half()  # coarse values: many exact ties
    if K > 3:
        x[:, 3] = x[:, 1]
    m = Guarded((B, 2 * H, 2 * W), torch.int64)
    from lseg_b200 import _lib
    from lseg_b200.ops import _ptr, _stream
    _lib.check(_lib.load().lseg_upsample2x_argmax(_ptr(x), _ptr(m.t), B, K, H, W, _stream()))
    m.check("upsample2x_argmax")
    assert torch.equal(m.t.cpu(), torch.max(ops.upsample2x_nchw(x).cpu(), 1)[1]), "upsample2x_argmax"


# ---------------------------------------------------------------------------------------------------------------
# L2 norms
# ---------------------------------------------------------------------------------------------------------------
def _l2_rows(M, C, seed, scale):
    x = _rand((M, C), seed, scale)
    x[0] = torch.where(_rand((C,), seed + 1) > 0, 1.0, -1.0)  # ||x||^2 = C exactly, whatever the order
    return x


@pytest.mark.parametrize("M,C", [(150, 512), (1, 512), (2, 256), (77 * 3, 512), (9, 768)])
def test_l2norm_f16(ops, M, C):
    x = _l2_rows(max(M, 1), C, 26, 0.3).half()
    y = Guarded((M, C), torch.float16)
    ops.l2norm_f16(x, out=y.t)
    y.check("l2norm_f16")
    _bound_ok(y.t, *G.l2norm_f16_ref(x), "l2norm_f16")
    emu = G.l2norm_f16_emulate(x)
    assert _bits_equal(y.t[0], emu[0]), "l2norm_f16: a row with an exact squared sum differs from the recipe"
    frac = G.bit_fraction(y.t, emu)
    assert frac >= 0.999, f"l2norm_f16: only {frac:.5f} of the elements match the float32 recipe bit for bit"


@pytest.mark.parametrize("M,C", [(1000, 512), (7, 128), (8 * 3600, 512), (33, 256), (5, 384)])
def test_l2norm_scale(ops, M, C):
    x = _l2_rows(M, C, 27, 2.0)
    y = Guarded((M, C), torch.float16)
    ops.l2norm_scale(x, LS, out=y.t)
    y.check("l2norm_scale")
    _bound_ok(y.t, *G.l2norm_scale_ref(x, LS), "l2norm_scale")
    emu = G.l2norm_scale_emulate(x, LS)
    assert _bits_equal(y.t[0], emu[0]), "l2norm_scale: a row with an exact squared sum differs from the recipe"
    frac = G.bit_fraction(y.t, emu)
    assert frac >= 0.999, f"l2norm_scale: only {frac:.5f} of the elements match the float32 recipe bit for bit"


# ---------------------------------------------------------------------------------------------------------------
# head blocks (arch_option 1 / 2)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("B,K,h,w", [(2, 7, 37, 56), (1, 3, 1, 1), (2, 5, 9, 33), (1, 2, 120, 120), (3, 21845, 1, 3)])
@pytest.mark.parametrize("mode,act", [(1, 2), (1, 0), (2, 3), (2, 1)])
def test_head_block(ops, B, K, h, w, mode, act, dtype):
    x = _rand((B, K, h, w), 28, 1.5, dtype)
    w9 = _rand((9,), 29, 0.3).tolist()
    y = Guarded((B, K, h, w), torch.float32)
    ops.head_block(x, w9, 0.17, mode, act, out=y.t)
    y.check("head_block")
    _bound_ok(y.t, *G.head_block_ref(x, w9, 0.17, mode, act), f"head_block mode {mode} act {act}")
    if B > 1:
        x2 = x.clone()
        x2[0] = 1.0
        assert _bits_equal(ops.head_block(x2, w9, 0.17, mode, act)[1:], y.t[1:]), "head_block: image independence"


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_channel_max_exact(ops, dtype):
    """With zero taps and bias, mode 1 returns the channel max itself: fmaf(0, x, 0) + 0 + cmax is exact."""
    x = _rand((3, 9, 13, 40), 30, 2.0, dtype)
    y = ops.head_block(x, [0.0] * 9, 0.0, 1, 0)
    assert _bits_equal(y, x.float().max(1, keepdim=True)[0].expand_as(y).contiguous()), "channel_max"


# ---------------------------------------------------------------------------------------------------------------
# text tower glue
# ---------------------------------------------------------------------------------------------------------------
def _tokens(K, L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.zeros((K, L), dtype=torch.int64)
    for k in range(K):
        n = int(torch.randint(0, L - 2, (1,), generator=g))
        t[k, 0] = 49406
        t[k, 1:1 + n] = torch.randint(1, 49406, (n,), generator=g)
        t[k, 1 + n] = 49407
        if k % 3 == 1 and n + 3 < L:
            t[k, n + 3] = 49407  # a second maximal id: the first one wins
    return t.cuda()


@pytest.mark.parametrize("K", [1, 5, 150, 129])
def test_text_embed_eot_gather_exact(ops, K):
    L, Wd = 77, 512
    tokens = _tokens(K, L, K)
    emb, pos = _rand((49408, Wd), 31, 0.02), _rand((L, Wd), 32, 0.01)
    x = Guarded((K * L, Wd), torch.float16)
    ops.text_embed(tokens, emb, pos, out=x.t)
    x.check("text_embed")
    ref = (emb[tokens].half() + pos.half()).view(K * L, Wd)
    assert _bits_equal(x.t, ref), "text_embed"
    rows = (K + 127) // 128 * 128
    out = Guarded((rows, Wd), torch.float16)
    ops.text_eot_gather(tokens, x.t, out=out.t)
    out.check("text_eot_gather")
    first = torch.tensor([int((row == row.max()).nonzero()[0]) for row in tokens.cpu()], device="cuda")
    assert _bits_equal(out.t[:K], x.t.view(K, L, Wd)[torch.arange(K, device="cuda"), first]), "text_eot_gather"
    assert bool((out.t[K:].view(torch.uint8) == SENT).all()), "text_eot_gather wrote into the padding rows"


# ---------------------------------------------------------------------------------------------------------------
# preprocess
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,Ho,Wo,Hp,Wp", [(1, 40, 3, 20, 3, 20), (37, 53, 480, 640, 480, 672), (480, 640, 240, 320,
                                                                                                    256, 320),
                                             (5, 5, 5, 5, 8, 9)])
def test_preprocess(ops, h, w, Ho, Wo, Hp, Wp):
    g = torch.Generator().manual_seed(h * w)
    img = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda()
    mean, std = (0.48, 0.46, 0.41), (0.27, 0.26, 0.28)
    out = Guarded((1, 3, Hp, Wp), torch.float32)
    ops.preprocess(img, (Ho, Wo), (Hp, Wp), mean, std, out=out.t)
    out.check("preprocess")
    # ToTensor then Normalize, each step one correctly rounded fp32 operation (formed in float64 and rounded once, which
    # is exact for + - / ; torch's CUDA division by a scalar multiplies by the reciprocal instead)
    m32 = torch.tensor(mean, dtype=torch.float32, device="cuda").double().view(3, 1, 1)
    s32 = torch.tensor(std, dtype=torch.float32, device="cuda").double().view(3, 1, 1)
    src = (img.permute(2, 0, 1).double() / 255).float()
    src = (src.double() - m32).float()
    src = (src.double() / s32).float()
    ref, absum, slack = G.bilinear_ref(src, Ho, Wo, False, contract_slack=True)
    ref, bound = G.bilinear_bound(ref, absum, slack)
    _bound_ok(out.t[0, :, :Ho, :Wo], ref, bound, "preprocess")
    pad = torch.tensor([-m / s for m, s in zip(mean, std)], dtype=torch.float32, device="cuda").view(3, 1, 1)
    full = pad.expand(3, Hp, Wp).clone()
    full[:, :Ho, :Wo] = out.t[0, :, :Ho, :Wo]
    assert _bits_equal(out.t[0], full), "preprocess padding"


# ---------------------------------------------------------------------------------------------------------------
# batch independence and determinism of the B-taking kernels
# ---------------------------------------------------------------------------------------------------------------
def _batch_cases(ops):
    yield "patchify", _rand((3, 3, 64, 96), 40), lambda x: ops.patchify(x).view(3, -1)
    yield "stem_im2col", _rand((3, 3, 16, 20), 41), lambda x: ops.stem_im2col(x).view(3, -1)
    yield "im2col_3x3_s2", _rand((3, 9, 7, 64), 42, dtype=torch.float16), lambda x: ops.im2col_3x3_s2(x).view(3, -1)
    yield "maxpool", _rand((3, 8, 6, 64), 43, dtype=torch.float16), ops.maxpool3x3s2_nhwc
    yield "subsample", _rand((3, 8, 6, 64), 44, dtype=torch.float16), ops.subsample2_nhwc
    yield "upsample2x_nhwc", _rand((3, 5, 7, 64), 45, dtype=torch.float16), ops.upsample2x_nhwc
    yield "readout_split", _rand((3, 10, 64), 46), lambda x: ops.readout_split(x)[0].view(3, -1)
    yield "assemble_tokens", _rand((3 * 9, 64), 47), \
        lambda x: ops.assemble_tokens(x, torch.ones(64, device="cuda"), torch.zeros((10, 64), device="cuda"), 3, 9)


def test_batch_independence_and_determinism(ops):
    for what, x, fn in _batch_cases(ops):
        y = fn(x)
        assert _bits_equal(fn(x), y), f"{what}: two runs differ"
        x2 = x.clone()
        x2.view(3, -1)[0] = -x2.view(3, -1)[0] - 1
        assert _bits_equal(fn(x2)[1:], y[1:]), f"{what}: images 1.. changed with image 0"


# ---------------------------------------------------------------------------------------------------------------
# engine glue: the fp32-input argmax behind the arch_option 1 head blocks at the smem line limit
# ---------------------------------------------------------------------------------------------------------------
def test_arch_option1_wide_image_predict_and_metric():
    """A 64x1024 image: the low-res logits are 512 wide (the smem line limit) and the 1024-wide output needs two
    512-column argmax passes of the fp32-input instantiation that runs after the head blocks."""
    from parity_util import NET_KW, synth
    from lseg_b200 import ops
    from lseg_b200.lseg_net import LSegNet
    from lseg_b200.metrics import SegmentationMetric
    sd = synth.make_state_dict(0, head_block=True)
    labels = synth.ade20k_labels()[:5]
    nk = dict(NET_KW)
    nk.update(arch_option=1, block_depth=2, activation="lrelu")
    net = LSegNet(labels=labels, **nk)
    net.load_state_dict(sd)
    net = net.cuda().eval()
    x = synth.make_image(1, 64, 1024, seed=7).cuda()
    tokens = synth.tokenize(labels)
    logits = net(x, tokens)
    mask = net.predict(x, tokens)
    assert torch.equal(mask, logits.argmax(1)), "predict() != forward().argmax(1)"
    g = torch.Generator().manual_seed(8)
    target = torch.randint(-1, 5, (1, 64, 1024), generator=g).cuda()
    metric = SegmentationMetric(5)
    net.update_metric(metric, x, target, tokens)
    want = torch.zeros((1, 3 * 5 + 2), dtype=torch.int64, device="cuda")
    ops.seg_stats_mask(mask, target, want, 5)
    assert torch.equal(metric.stats, want), "update_metric != seg_stats_mask(predict())"


# ---------------------------------------------------------------------------------------------------------------
# argument validation: each rejection names the entry and the argument, launches nothing, leaves outputs untouched
# ---------------------------------------------------------------------------------------------------------------
def _p(t, off=0):
    return C.c_void_p(t.data_ptr() + off) if t is not None else None


def _reject(fn_name, args, out, entry, arg):
    from lseg_b200 import _lib
    from lseg_b200.ops import _stream
    rc = getattr(_lib.load(), fn_name)(*args, _stream())
    torch.cuda.synchronize()
    assert rc != 0, f"{fn_name} accepted a bad {arg}"
    msg = _lib.load().lseg_last_error().decode()
    # the argument must be the subject of the message: right after the entry prefix (or "null "), as a whole word
    named = msg.startswith(entry + ":") and re.match(rf"{re.escape(entry)}: (null )?{re.escape(arg)}(?![\w*(/])", msg)
    assert named, f"{fn_name}: error {msg!r} does not name {entry} / {arg}"
    out.check(f"{fn_name} rejection")
    assert bool((out.t.view(torch.uint8) == SENT).all()), f"{fn_name}: output written before the rejection"


F16, F32, I64 = torch.float16, torch.float32, torch.int64
W9, M3, S3 = (lambda: (C.c_float * 9)()), (lambda: (C.c_float * 3)()), (lambda: (C.c_float * 3)(1, 1, 1))

# (entry, argument, output shape, output dtype, args given the output o and the input buffers b: x32 / x16 / tok)
REJECTIONS = [
    ("lseg_layernorm", "M", (8, 512), F16,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(b.x32), _p(o), C.c_longlong(0), 512, C.c_float(1e-6))),
    ("lseg_layernorm", "gamma", (8, 512), F16,
     lambda o, b: (_p(b.x32), 0, _p(b.x32, 4), _p(b.x32), _p(o), C.c_longlong(8), 512, C.c_float(1e-6))),
    ("lseg_layernorm", "y", (8, 512), F16,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(b.x32), _p(o, 2), C.c_longlong(1), 512, C.c_float(1e-6))),
    ("lseg_patchify", "x", (4, 768), F16, lambda o, b: (None, _p(o), 1, 32, 32, 16)),
    ("lseg_patchify", "B*(H/patch)", (4, 768), F16, lambda o, b: (_p(b.x32), _p(o), 65536, 16, 16, 16)),
    ("lseg_pos_resize", "gh", (4, 8), F32, lambda o, b: (_p(b.x32), _p(o), 4, 0, 2, 8)),
    ("lseg_pos_resize", "out", (4, 8), F32, lambda o, b: (_p(b.x32), None, 4, 1, 2, 8)),
    ("lseg_assemble_tokens", "D", (2, 6), F32, lambda o, b: (_p(b.x32), _p(b.x32), _p(b.x32), _p(o), 1, 1, 6)),
    ("lseg_assemble_tokens", "patch", (2, 8), F32, lambda o, b: (_p(b.x32, 4), _p(b.x32), _p(b.x32), _p(o), 1, 1, 8)),
    ("lseg_readout_split", "D", (2, 6), F16, lambda o, b: (_p(b.x32), _p(o), _p(o), 1, 1, 6)),
    ("lseg_readout_split", "T", (2, 8), F16, lambda o, b: (_p(b.x32), _p(o), _p(o), 1, -1, 8)),
    ("lseg_im2col_3x3_s2", "C", (4, 9 * 12), F16, lambda o, b: (_p(b.x16), _p(o), 1, 3, 3, 12)),
    ("lseg_im2col_3x3_s2", "a", (4, 9 * 8), F16, lambda o, b: (_p(b.x16), _p(o, 2), 1, 3, 3, 8)),
    ("lseg_im2col_3x3_s2", "B", (4, 9 * 8), F16, lambda o, b: (_p(b.x16), _p(o), 65536, 3, 3, 8)),
    ("lseg_stem_im2col", "B*(H/2)*(W/2)", (4, 192), F16, lambda o, b: (_p(b.x32), _p(o), 65536, 1024, 1024)),
    ("lseg_stem_im2col", "H", (4, 192), F16, lambda o, b: (_p(b.x32), _p(o), 1, 0, 4)),
    ("lseg_maxpool3x3s2_nhwc", "B", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16), _p(o), 65536, 2, 2, 8)),
    ("lseg_maxpool3x3s2_nhwc", "x", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16, 8), _p(o), 1, 2, 2, 8)),
    ("lseg_subsample2_nhwc", "B", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16), _p(o), 65536, 2, 2, 8)),
    ("lseg_subsample2_nhwc", "y", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16), None, 1, 2, 2, 8)),
    ("lseg_upsample2x_nhwc", "C", (1, 2, 2, 12), F16, lambda o, b: (_p(b.x16), _p(o), 1, 1, 1, 12)),
    ("lseg_upsample2x_nhwc", "2H", (1, 2, 2, 8), F16, lambda o, b: (_p(b.x16), _p(o), 1, 40000, 1, 8)),
    ("lseg_upsample2x_nhwc256", "add", (1, 2, 2, 256), F32,
     lambda o, b: (_p(b.x16), 1, _p(o), 0, _p(b.x32, 4), 1, 1, 1)),
    ("lseg_upsample2x_nhwc256", "B", (1, 2, 2, 256), F32, lambda o, b: (_p(b.x16), 1, _p(o), 0, None, 65536, 1, 1)),
    ("lseg_l2norm_scale", "M", (1, 128), F16, lambda o, b: (_p(b.x32), _p(o), C.c_longlong(0), 128, C.c_float(1.0))),
    ("lseg_l2norm_scale", "x", (1, 128), F16, lambda o, b: (_p(b.x32, 4), _p(o), C.c_longlong(1), 128, C.c_float(1.0))),
    ("lseg_l2norm_f16", "C", (1, 8), F16, lambda o, b: (_p(b.x16), _p(o), 1, 0)),
    ("lseg_l2norm_f16", "y", (1, 8), F16, lambda o, b: (_p(b.x16), _p(o, 1), 1, 8)),
    ("lseg_upsample2x_nchw", "planes", (1, 2, 16), F32, lambda o, b: (_p(b.x16), _p(o), C.c_longlong(0), 1, 8)),
    ("lseg_upsample2x_nchw", "x", (1, 2, 16), F32, lambda o, b: (_p(b.x16, 2), _p(o), C.c_longlong(1), 1, 8)),
    ("lseg_upsample2x_nchw_bg", "H", (1, 2, 16), F32, lambda o, b: (_p(b.x16), _p(o), C.c_longlong(1), 0, 8)),
    ("lseg_upsample2x_nchw_f32", "y", (1, 2, 16), F32, lambda o, b: (_p(b.x32), _p(o, 4), C.c_longlong(1), 1, 8)),
    ("lseg_head_block", "cmax_ws", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, None, _p(o), 1, 1, 4, 4, W9(), C.c_float(0), 1, 0)),
    ("lseg_head_block", "mode", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(o), 1, 1, 4, 4, W9(), C.c_float(0), 3, 0)),
    ("lseg_head_block", "K", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(o), 1, 0, 4, 4, W9(), C.c_float(0), 2, 0)),
    ("lseg_text_embed", "tokens", (2, 8), F16, lambda o, b: (_p(b.tok, 4), _p(b.x32), _p(b.x32), _p(o), 1, 2, 8)),
    ("lseg_text_embed", "L", (2, 8), F16, lambda o, b: (_p(b.tok), _p(b.x32), _p(b.x32), _p(o), 1, 0, 8)),
    ("lseg_text_eot_gather", "K", (128, 8), F16, lambda o, b: (_p(b.tok), _p(b.x16), _p(o), 0, 2, 8)),
    ("lseg_text_eot_gather", "out", (128, 8), F16, lambda o, b: (_p(b.tok), _p(b.x16), None, 1, 2, 8)),
    ("lseg_preprocess", "Hp", (1, 3, 4, 4), F32,
     lambda o, b: (_p(b.u8), _p(o), 4, 4, 4, 4, 3, 4, M3(), S3(), M3())),
    ("lseg_preprocess", "img_hwc", (1, 3, 4, 4), F32,
     lambda o, b: (None, _p(o), 4, 4, 4, 4, 4, 4, M3(), S3(), M3())),
    # shape rules and grid limits
    ("lseg_layernorm", "C", (8, 512), F16,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(b.x32), _p(o), C.c_longlong(1), 256, C.c_float(1e-6))),
    ("lseg_patchify", "patch", (4, 768), F16, lambda o, b: (_p(b.x32), _p(o), 1, 16, 16, 8)),
    ("lseg_patchify", "W", (4, 768), F16, lambda o, b: (_p(b.x32), _p(o), 1, 16, 24, 16)),
    ("lseg_stem_im2col", "W", (4, 192), F16, lambda o, b: (_p(b.x32), _p(o), 1, 4, 5)),
    ("lseg_maxpool3x3s2_nhwc", "C", (1, 1, 1, 12), F16, lambda o, b: (_p(b.x16), _p(o), 1, 2, 2, 12)),
    ("lseg_maxpool3x3s2_nhwc", "H", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16), _p(o), 1, 3, 2, 8)),
    ("lseg_subsample2_nhwc", "W", (1, 1, 1, 8), F16, lambda o, b: (_p(b.x16), _p(o), 1, 2, 3, 8)),
    ("lseg_im2col_3x3_s2", "Ho", (4, 9 * 8), F16, lambda o, b: (_p(b.x16), _p(o), 1, 131072, 1, 8)),
    ("lseg_upsample2x_nhwc256", "add", (1, 2, 2, 256), F16,
     lambda o, b: (_p(b.x16), 1, _p(o), 1, _p(b.x32), 1, 1, 1)),
    ("lseg_l2norm_scale", "C", (1, 64), F16, lambda o, b: (_p(b.x32), _p(o), C.c_longlong(1), 64, C.c_float(1.0))),
    ("lseg_upsample2x_nchw", "W", (1, 2, 24), F32, lambda o, b: (_p(b.x16), _p(o), C.c_longlong(1), 1, 12)),
    ("lseg_upsample2x_nchw", "planes", (1, 2, 16), F32, lambda o, b: (_p(b.x16), _p(o), C.c_longlong(65536), 1, 8)),
    ("lseg_upsample2x_nchw_f32", "W", (1, 2, 16), F32, lambda o, b: (_p(b.x32), _p(o), C.c_longlong(1), 1, 520)),
    ("lseg_upsample2x_nchw_bg", "W", (1, 2, 6), F32, lambda o, b: (_p(b.x16), _p(o), C.c_longlong(1), 1, 3)),
    ("lseg_upsample2x_argmax", "W", (1, 2, 24), I64, lambda o, b: (_p(b.x16), _p(o), 1, 2, 1, 12)),
    ("lseg_upsample2x_argmax", "mask", (1, 2, 16), I64, lambda o, b: (_p(b.x16), _p(o, 4), 1, 2, 1, 8)),
    ("lseg_head_block", "act", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(o), 1, 1, 4, 4, W9(), C.c_float(0), 2, 4)),
    ("lseg_head_block", "ceil(h/8)", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(o), 1, 1, 8 * 65536, 1, W9(), C.c_float(0), 2, 0)),
    ("lseg_head_block", "B*K", (1, 1, 4, 4), F32,
     lambda o, b: (_p(b.x32), 0, _p(b.x32), _p(o), 2, 40000, 1, 1, W9(), C.c_float(0), 2, 0)),
    ("lseg_text_embed", "K*L", (2, 8), F16, lambda o, b: (_p(b.tok), _p(b.x32), _p(b.x32), _p(o), 65536, 65536, 8)),
    ("lseg_preprocess", "ceil(Hp/8)", (1, 3, 4, 4), F32,
     lambda o, b: (_p(b.u8), _p(o), 4, 4, 4, 4, 8 * 65536, 4, M3(), S3(), M3())),
]


class _Inputs:
    def __init__(self):
        self.x32 = torch.zeros(4096, dtype=F32, device="cuda")
        self.x16 = torch.zeros(4096, dtype=F16, device="cuda")
        self.tok = torch.zeros(64, dtype=I64, device="cuda")
        self.u8 = torch.zeros(4096, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("entry,arg,shape,dtype,build", REJECTIONS, ids=[f"{e}-{a}" for e, a, *_ in REJECTIONS])
def test_rejects_bad_arguments(ops, entry, arg, shape, dtype, build):
    out = Guarded(shape, dtype)
    out.t.view(torch.uint8).fill_(SENT)
    _reject(entry, build(out.t, _Inputs()), out, entry, arg)


@pytest.mark.parametrize("what", ["dtype", "shape", "strided"])
def test_out_validation(ops, what):
    from lseg_b200 import _lib
    x = _rand((8, 512), 50)
    g = _rand((512,), 51)
    out = {"dtype": torch.empty((8, 512), dtype=torch.float32, device="cuda"),
           "shape": torch.empty((8, 513), dtype=torch.float16, device="cuda"),
           "strided": torch.empty((512, 8), dtype=torch.float16, device="cuda").t()}[what]
    with pytest.raises(_lib.LsegError, match="layernorm: out must be"):
        ops.layernorm(x, g, g, 1e-6, out=out)
