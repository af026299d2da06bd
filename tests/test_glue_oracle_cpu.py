"""The glue-kernel bounds of tests/glue_oracle.py are neither too loose nor too tight: on CPU, a float32 emulation of each
kernel's recipe passes its oracle, and a fake kernel with one planted defect fails it."""
import math

import pytest
import torch

import glue_oracle as G

LS = math.exp(math.log(1 / 0.07))


def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64) * scale


def _ln_inputs(C, dtype, seed):
    """Rows with ordinary statistics, |mean| >> std, variance near eps, and a constant row."""
    x = _randn((64, C), seed, 2.0)
    x[1] = 300.0 + _randn((C,), seed + 1, 0.05)[:]
    x[2] = 0.5 + _randn((C,), seed + 2, 1e-3)
    x[3] = 7.0
    x = x.to(dtype)
    g = _randn((C,), seed + 3).float()
    b = _randn((C,), seed + 4, 0.1).float()
    return x, g, b


@pytest.mark.parametrize("C", [512, 768, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_layernorm_emulation_passes(C, dtype):
    x, g, b = _ln_inputs(C, dtype, C)
    eps = 1e-5 if dtype == torch.float16 else 1e-6
    ref, bound = G.layernorm_ref(x, g, b, eps)
    n, msg = G.violations(G.layernorm_emulate(x, g, b, eps), ref, bound)
    assert n == 0, msg


@pytest.mark.parametrize("defect", ["no_eps", "ddof1"])
def test_layernorm_defects_caught(defect):
    x, g, b = _ln_inputs(512, torch.float32, 5)
    eps = 1e-6
    ref, bound = G.layernorm_ref(x, g, b, eps)
    bad = G.layernorm_emulate(x, g, b, eps, use_eps=defect != "no_eps", ddof=1 if defect == "ddof1" else 0)
    n, _ = G.violations(bad, ref, bound)
    assert n > 0, f"layernorm defect {defect} not caught"


@pytest.mark.parametrize("shape", [(2, 3, 1, 1), (1, 2, 3, 17), (2, 4, 15, 33), (1, 1, 23, 8)])
def test_upsample_emulation_passes_and_swap_caught(shape):
    x = _randn(shape, 11, 3.0).float()
    ref, bound = G.upsample2x_ref(x)
    n, msg = G.violations(G.upsample2x_emulate(x), ref, bound)
    assert n == 0, msg
    ref16, bound16 = G.upsample2x_ref(x, out_f16=True)
    n, msg = G.violations(G.upsample2x_emulate(x).half(), ref16, bound16)
    assert n == 0, msg
    if shape[-1] > 1:  # W = 1 has lx = 0 everywhere: swapping the weights of one tap is no defect there
        n, _ = G.violations(G.upsample2x_emulate(x, swap_x=True), ref, bound)
        assert n > 0, "upsample with hx / lx swapped not caught"


@pytest.mark.parametrize("g0,gh,gw", [(24, 30, 46), (24, 4, 6), (12, 15, 23)])
def test_half_pixel_bilinear_emulation_passes(g0, gh, gw):
    """The align_corners=False resize (pos_resize, preprocess) with ATen's rounded coordinate product passes, and so does
    the same product contracted into an FMA (emulated by forming the coordinate in float64 and rounding once)."""
    x = _randn((8, g0, g0), 12).float()
    ref, absum, slack = G.bilinear_ref(x, gh, gw, False, contract_slack=True)
    _, bound = G.bilinear_bound(ref, absum, slack)
    for fma in (False, True):
        def coords(n_in, n_out):
            dst = torch.arange(n_out, dtype=torch.float64)
            s = torch.tensor(float(n_in), dtype=torch.float32) / float(n_out)
            if fma:
                src = (s.double() * (dst + 0.5) - 0.5).float().clamp_min(0)
            else:
                src = (s * (dst.float() + 0.5) - 0.5).clamp_min(0)
            i0 = src.long().clamp_max(n_in - 1)
            i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
            l1 = src - i0.float()
            return i0, i1, 1.0 - l1, l1
        y0, y1, hy, ly = coords(g0, gh)
        x0, x1, hx, lx = coords(g0, gw)
        r0, r1 = x[:, y0, :], x[:, y1, :]
        hy, ly = hy[:, None], ly[:, None]
        got = hy * (hx * r0[..., x0] + lx * r0[..., x1]) + ly * (hx * r1[..., x0] + lx * r1[..., x1])
        n, msg = G.violations(got, ref, bound)
        assert n == 0, f"fma={fma}: {msg}"


def _l2_rows(C, seed):
    x = _randn((400, C), seed, 0.3)
    x[0] = torch.where(_randn((C,), seed + 1) > 0, 1.0, -1.0)  # ||x||^2 = C exactly, in any order
    return x


@pytest.mark.parametrize("C", [512, 768])
def test_l2norm_f16_emulation_passes_and_defect_caught(C):
    x = _l2_rows(C, 13).half()
    ref, bound = G.l2norm_f16_ref(x)
    good = G.l2norm_f16_emulate(x)
    assert G.violations(good, ref, bound)[0] == 0
    bad = G.l2norm_f16_emulate(x, round_norm=False)
    # a missing fp16 rounding of the norm stays within one norm ulp: the bit-level contract is what catches it
    assert G.bit_fraction(bad, good) < 0.999, "l2norm_f16 without the fp16 norm rounding not caught"


@pytest.mark.parametrize("C", [128, 512])
def test_l2norm_scale_emulation_passes_and_defect_caught(C):
    x = _l2_rows(C, 14).float()
    ref, bound = G.l2norm_scale_ref(x, LS)
    good = G.l2norm_scale_emulate(x, LS)
    assert G.violations(good, ref, bound)[0] == 0
    bad = G.l2norm_scale_emulate(x, LS, scale_first=True)
    assert G.bit_fraction(bad, good) < 0.999, "l2norm_scale with logit_scale applied before rounding not caught"


@pytest.mark.parametrize("mode,act", [(1, 0), (1, 1), (1, 2), (1, 3), (2, 0), (2, 1), (2, 2), (2, 3)])
def test_head_block_emulation_passes(mode, act):
    x = _randn((2, 5, 13, 37), 15, 1.5).float()
    w9 = _randn((9,), 16, 0.3).float().tolist()
    ref, bound = G.head_block_ref(x, w9, 0.17, mode, act)
    n, msg = G.violations(G.head_block_emulate(x, w9, 0.17, mode, act), ref, bound)
    assert n == 0, msg


@pytest.mark.parametrize("act", [1, 2, 3])
def test_head_block_act_before_cmax_caught(act):
    x = _randn((2, 5, 13, 37), 17, 1.5).float()
    w9 = _randn((9,), 18, 0.3).float().tolist()
    ref, bound = G.head_block_ref(x, w9, -0.3, 1, act)
    n, _ = G.violations(G.head_block_emulate(x, w9, -0.3, 1, act, act_before_cmax=True), ref, bound)
    assert n > 0, f"head_block act {act} applied before the cmax add not caught"
