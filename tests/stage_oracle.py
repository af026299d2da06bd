"""Float64 references and error bounds for the stages of the engine's image path (csrc/engine.cuh, build_vit_trunk and
build_image_plan: readout -> reassemble -> layer_rn -> fusion decoder -> head1 -> pixel x text), each stage fed the
engine's own input of that stage, plus float32 emulations of the engine's recipe with planted defects.

Shared by tests/test_image_stages_gpu.py (against the stage buffers of one engine forward, `Engine.debug_tensor`) and
tests/test_image_stages_cpu.py (the emulations must pass, every planted defect must fail). Plain torch: CPU or CUDA.
Decoder tensors are NHWC; weights are the state dict's, rounded to fp16 where packing.py rounds them; eval BatchNorm is
folded to an fp32 scale and shift as packing.fold_bn folds it. Each reference is the reference module's math (e.g.
out_conv after the x2 interpolation), so a bound that holds also shows the engine's reordering to be legitimate.

Bounds (u = 2^-24; u_tc = 2^-23, tensor-core fp32 accumulation charged a full ulp per addition as in
attention_oracle.py; gamma_n = n u_tc / (1 - n u_tc); mag = sum |a| |w| over the n terms of an output):

    accumulate        fp16 operands, products exact in fp32          gamma_n mag
    scale, bias       v * s + b (two roundings, or one FMA)          |s| acc_err + 2 u (|s| mag + |b|)
    relu              1-Lipschitz                                     unchanged
    gelu              gelu_erf (common.cuh): 3.7e-6 + 2^-21 |x|       1.13 err + 3.7e-6 + 2^-21 (|x| + err)
                      (1.13 >= max |gelu'| = 1.129)
    residual add      one fp32 add per operand                        + u (|y| + err)
    fp16 store        round to nearest                                + ulp16(|y| + err) / 2

An operand the stage cannot observe (readout -> post for levels 0-2, RCU1's conv1 output) enters through its own bound
e_in: the next product adds sum |w| e_in to the error and to mag. For such a stage the tier-B reference (`ref_b`) applies
the intermediate's fp16 rounding in float64 (rn16 of the float64 intermediate), which is what the engine rounds.

Interpolation (dec{k}_skip, path1, the arch_option output): glue_oracle.upsample2x_ref, with the interpolated operand's
own bound carried through the (non-negative, sum-to-one) interpolation weights.

head1's partial squared norms (feat_sumsq[p, j] = sum over columns 32 j .. 32 j + 31 of f^2, f the fp32 pre-rounding
head1 output, one fmaf chain): |S' - S| <= sum (2 |f| e + e^2) + gamma_32(u) sum (|f| + e)^2, e = f's fp32 bound.

pixel x text (one logit = rn16(logit_scale * rsqrtf(sum of the row's parts) * (featn . text))):
    dot               gamma_C sum |f| |t|
    norm              parts summed in fp32 (n_parts adds), rsqrtf 2 ulp, two products: relative
                      rel = gamma_np(u) / 2 + 2^-22 + 2 u (+ second order, absorbed by doubling the total)

Tiers. A: every element within the bound. B (sensitivity): fp16 outputs must be bit-identical to rn16(ref_b) on at least
FP16_IDENTICAL of their elements (for the readout, of those with |GELU| >= 2^-7, where gelu_erf is documented accurate
to half an fp16 ulp; FP16_IDENTICAL_CHAINED for post{k}, k < 3, whose operand is the unobservable fp16 readout: gelu_erf's
error moves a few percent of that readout's fp16 roundings to the neighbouring value, and with ~1000 terms per output
each moved term shifts the output by |w| fp16 ulps of the readout, so rn16(ref_b) is only the likeliest output); fp32 outputs must have an RMS error below FP32_RMS x the RMS half fp16 ulp of the
output (no hidden fp16 rounding). Both thresholds are fixed by tests/test_image_stages_cpu.py: the float32 emulation of
every stage clears them and the planted sub-ulp defects do not.
"""
import math

import torch
import torch.nn.functional as F

import glue_oracle as G
from glue_oracle import U, r16, ulp16

UTC = 2.0 ** -23
GELU_LIP = 1.13
FP16_IDENTICAL = 0.95
FP16_IDENTICAL_CHAINED = 0.75  # post{k}, k < 3: through the unobservable fp16 GELU readout (module docstring)
FP32_RMS = 0.1
F64 = torch.float64


def gamma(n, u=UTC):
    return n * u / (1 - n * u)


def w16(w):
    """A weight as packing.py stores it: rounded to fp16."""
    return r16(w.to(F64))


def fold_bn(sd, prefix, eps=1e-5):
    """packing.fold_bn's fp32 (scale, shift), as float64."""
    from lseg_b200.packing import fold_bn as fold
    s, t = fold(sd, prefix, eps)
    return s.double(), t.double()


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _dev(t, like):
    return t.to(device=like.device, dtype=F64)


# ------------------------------------------------------------------------------------------------------------------
# generic: products, epilogue
# ------------------------------------------------------------------------------------------------------------------
def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def conv_terms(x, w, *, stride=1, pad=1, e_in=None, transpose=False):
    """x NHWC values, w [Cout, Cin, kh, kw] (ConvTranspose: [Cin, Cout, s, s], stride s) -> (acc, mag, n) NHWC float64;
    e_in: the operand's own bound (NHWC), carried through |w| into acc's error and mag."""
    x = _nchw(x.to(F64))
    w = w.to(device=x.device, dtype=F64)
    op = ((lambda a, b: F.conv_transpose2d(a, b, stride=stride)) if transpose else
          (lambda a, b: F.conv2d(a, b, stride=stride, padding=pad)))
    acc = op(x, w)
    mag = op(x.abs(), w.abs())
    prop = None
    if e_in is not None:
        prop = _nhwc(op(_nchw(e_in.to(F64)), w.abs()))
    n = w.shape[0] if transpose else w[0].numel()
    return _nhwc(acc), _nhwc(mag), n, prop


def linear_terms(x, w, e_in=None):
    """x [M, K] values, w [N, K] -> (acc, mag, n, prop)."""
    x = x.to(F64)
    w = w.to(device=x.device, dtype=F64)
    prop = e_in.to(F64) @ w.abs().t() if e_in is not None else None
    return x @ w.t(), x.abs() @ w.abs().t(), w.shape[1], prop


def epilogue(acc, mag, n, prop=None, *, scale=None, bias=None, act=None, res=(), out_f16=False):
    """float64 (ref, bound) of act(acc * scale + bias) + sum(res), rounded to fp16 when out_f16 (module docstring)."""
    if prop is None:
        prop = torch.zeros_like(acc)
    E = gamma(n) * (mag + prop) + prop
    m = mag + prop
    y = acc
    if scale is not None:
        s = _dev(scale, acc)
        y, E, m = y * s, E * s.abs(), m * s.abs()
    if bias is not None:
        b = _dev(bias, acc)
        y = y + b
        E = E + 2 * U * (m + b.abs())
    elif scale is not None:
        E = E + 2 * U * m
    if act == "relu":
        y = y.clamp_min(0)
    elif act == "gelu":
        E = GELU_LIP * E + 3.7e-6 + 2.0 ** -21 * (y.abs() + E)
        y = gelu64(y)
    for r in res:
        y = y + r.to(F64)
        E = E + U * (y.abs() + E)
    if out_f16:
        E = E + ulp16(y.abs() + E) / 2
    return y, E


# ------------------------------------------------------------------------------------------------------------------
# stages
# ------------------------------------------------------------------------------------------------------------------
def readout(tap, w, b):
    """ProjectReadout (GELU(Linear(cat(tok, cls)))) of tap fp32 [B, 1 + T, D] -> [B*T, D]: readout_split rounds the tap
    to fp16 (tested bit-exact in test_glue_gpu.py), so the float64 reference takes rn16(tap) as its operand."""
    x = r16(tap.to(F64))
    B, N, D = x.shape
    tok, cls = x[:, 1:], x[:, 0]
    wt, wc = w16(w[:, :D]).to(x.device), w16(w[:, D:]).to(x.device)
    acc = tok @ wt.t() + (cls @ wc.t())[:, None]
    mag = tok.abs() @ wt.abs().t() + (cls.abs() @ wc.abs().t())[:, None]
    ref, E = epilogue(acc.reshape(B * (N - 1), -1), mag.reshape(B * (N - 1), -1), D, bias=b, act="gelu",
                      out_f16=True)
    # tier B counts the outputs where gelu_erf's error is documented below half an fp16 ulp (|gelu| >= 2^-7)
    return {"ref": ref, "bound": E, "b_mask": ref.abs() >= 2.0 ** -7}


def post(ro, w, b, e_in=None):
    """act_postprocess 1x1 conv of the readout rows [B*T, D] -> fp16 [B*T, c]; w [c, D, 1, 1], zero-padded by the caller
    to the stored channel count. e_in: ro's bound when ro is the float64 readout reference (the fp16 readout of levels
    0-2 is not observable)."""
    wk = w16(w.reshape(w.shape[0], -1))
    acc, mag, n, prop = linear_terms(ro, wk, e_in)
    ref, E = epilogue(acc, mag, n, prop, bias=b, out_f16=True)
    out = {"ref": ref, "bound": E}
    if e_in is not None:
        out["ref_b"] = r16(ro.to(F64)) @ _dev(wk, ref).t() + _dev(b, ref)
        out["b_min"] = FP16_IDENTICAL_CHAINED
    return out


def resample(x, r, w, b):
    """Reassemble resample of post{k} NHWC [B, gh, gw, c] -> layer{k}, fp16: r > 0 ConvTranspose2d (kernel = stride = r),
    r = -2 Conv2d 3x3 stride 2 pad 1. Weights and bias zero-padded to the stored channels by the caller."""
    if r > 0:
        acc, mag, n, prop = conv_terms(x, w16(w), stride=r, transpose=True)
    else:
        acc, mag, n, prop = conv_terms(x, w16(w), stride=2, pad=1)
    ref, E = epilogue(acc, mag, n, prop, bias=b, out_f16=True)
    return {"ref": ref, "bound": E}


def conv3x3(x, w, *, scale=None, shift=None, act=None, res=(), out_f16=False, e_in=None):
    """A 3x3 stride-1 pad-1 conv of the decoder (layer_rn, the RCU convs) on NHWC x, epilogue as the engine's."""
    acc, mag, n, prop = conv_terms(x, w16(w), e_in=e_in)
    ref, E = epilogue(acc, mag, n, prop, scale=scale, bias=shift, act=act, res=res, out_f16=out_f16)
    return {"ref": ref, "bound": E}


def rcu1(x_relu, skip, w1, bn1, w2, bn2):
    """output = xs[0] + resConfUnit1(xs[1]), fed xs[1]'s ReLU'd fp16 copy x_relu (rn{k}_relu) and xs[0] + xs[1] already
    summed into the fp32 skip (dec{k+1}_skip): bn2(conv2(relu(bn1(conv1(x_relu))))) + skip, fp32. The conv1 output (fp16)
    is not observable: its bound is carried through |w2|."""
    h = conv3x3(x_relu, w1, scale=bn1[0], shift=bn1[1], act="relu", out_f16=True)
    out = conv3x3(h["ref"], w2, scale=bn2[0], shift=bn2[1], res=(skip,), e_in=h["bound"])
    acc_b = conv_terms(r16(h["ref"]), w16(w2))[0]
    out["ref_b"] = acc_b * _dev(bn2[0], acc_b) + _dev(bn2[1], acc_b) + skip.to(F64)
    return out


def out_conv(x, w, b, *, out_f16=False):
    """refinenet out_conv (1x1 + bias) on the low-res RCU2 output NHWC: fp32, or fp16 under LSEG_OUTCONV_F16."""
    acc, mag, n, prop = conv_terms(x, w16(w), pad=0)
    ref, E = epilogue(acc, mag, n, prop, bias=b, out_f16=out_f16)
    return {"ref": ref, "bound": E}


def _up(x):
    """bilinear x2 align_corners=True of NCHW float64 x with ATen's fp32 weights -> (value, sum |w_i v_i|)."""
    ref, absum, _ = G.bilinear_ref(x, 2 * x.shape[-2], 2 * x.shape[-1], True)
    return ref, absum


def upsample_skip(x, add=None, *, out_f16=False, e_in=None):
    """bilinear x2 (align_corners=True) of NHWC x, + the next level's fp32 layer_rn output `add` -> NHWC (dec{k}_skip,
    or path1 in fp16 at level 0). e_in: x's own bound when x is a float64 reference, carried through the weights."""
    xc = _nchw(x.to(F64))
    ref, absum = _up(xc)
    carried = 0.0
    if e_in is not None:
        absum = _up(xc.abs() + _nchw(e_in))[0]
        carried = _up(_nchw(e_in.to(F64)))[0]
    ref, E = G.bilinear_bound(ref, absum, add=None if add is None else _nchw(add))
    E = E + carried
    if out_f16:
        E = E + ulp16(ref.abs() + E) / 2
    return {"ref": _nhwc(ref), "bound": _nhwc(E)}


def out_conv_upsampled(x, w, b, add=None, *, lr_f16=False, out_f16=False):
    """The fusion block's tail as the reference module computes it, interpolate(x2) THEN out_conv, on the low-res RCU2
    output NHWC x, + `add`: the engine's conv-then-interpolate order is legitimate iff its output is inside this bound.
    The interpolation weights sum to one up to 2 u (fp32(1 - lambda) + lambda), which moves the bias by 2 u |b|."""
    xc = _nchw(x.to(F64))
    up, _ = _up(xc)
    oc = out_conv(x, w, b, out_f16=lr_f16)
    wk = _dev(w16(w), up)
    ref = F.conv2d(up, wk, _dev(b, up))
    absum = _up(_nchw(oc["ref"].abs() + oc["bound"]))[0]
    carried = _up(_nchw(oc["bound"]))[0]
    ref, E = G.bilinear_bound(ref, absum, add=None if add is None else _nchw(add))
    E = E + carried + 2 * U * _dev(b, up).abs().view(1, -1, 1, 1)
    if out_f16:
        E = E + ulp16(ref.abs() + E) / 2
    out = {"ref": _nhwc(ref), "bound": _nhwc(E)}
    if lr_f16:  # tier B: the low-res result rounded to fp16 where the engine rounds it
        ref_b = _up(_nchw(r16(oc["ref"])))[0]
        out["ref_b"] = _nhwc(ref_b if add is None else ref_b + _nchw(add).to(F64))
    return out


def head1(p1, w, b):
    """scratch.head1 (1x1 conv + bias) on path1 NHWC [B, h, w, 256] -> featn fp16 [.., out_c] and feat_sumsq fp32
    [.., out_c / 32] (squares of the fp32 pre-rounding output, per 32-column chunk)."""
    acc, mag, n, _ = conv_terms(p1, w16(w), pad=0)
    f, Ef = epilogue(acc, mag, n, bias=b)
    featn = {"ref": f, "bound": Ef + ulp16(f.abs() + Ef) / 2}
    chunks = f.shape[:-1] + (f.shape[-1] // 32, 32)
    fa, ea = f.abs().reshape(chunks), Ef.reshape(chunks)
    S = (fa * fa).sum(-1)
    ES = (2 * fa * ea + ea * ea).sum(-1) + gamma(32, U) * ((fa + ea) ** 2).sum(-1)
    return featn, {"ref": S, "bound": ES}


def pixel_text(featn, sumsq, text, K, logit_scale, stride=0):
    """logits_lr [B, K, P] of featn [B, P, C] (fp16 values), sumsq [B, P, C/32] and text rows [rows, C]: image b uses
    rows [b * stride, b * stride + K) (the zero-shot per-image blocks), or rows [0, K) when stride == 0.
    ref = logit_scale * (f . t) / sqrt(sum of the row's parts)."""
    f = featn.to(F64)
    B, P, C = f.shape
    ls = float(torch.tensor(logit_scale, dtype=torch.float32))
    S = sumsq.to(F64).sum(-1, keepdim=True)
    scale = ls / torch.sqrt(S)
    rel = gamma(sumsq.shape[-1], U) / 2 + 2.0 ** -22 + 2 * U
    refs, bounds = [], []
    for b in range(B):
        t = text[b * stride:b * stride + K] if stride else text[:K]
        t = _dev(t, f)
        dot, mag = f[b] @ t.t(), f[b].abs() @ t.abs().t()
        ref = scale[b] * dot
        E = 2 * scale[b] * (gamma(C) * mag + dot.abs() * rel)
        E = E + ulp16(ref.abs() + E) / 2
        refs.append(ref.t())
        bounds.append(E.t())
    return {"ref": torch.stack(refs), "bound": torch.stack(bounds)}


def head_blocks(lr, w9, bias, mode, act, depth):
    """scratch.head_block applied as lseg_net.py:198-201 (depth - 1 times with the activation, once without) on the fp16
    low-res logits NCHW, then the x2 output interpolation -> fp32 logits NCHW. The fp32 block outputs in between are not
    observable: each block's bound is carried through the next one's |taps| (and, for mode 1, its channel max)."""
    x, E = lr.to(F64), torch.zeros_like(lr, dtype=F64)
    for d in range(depth):
        a = act if d + 1 < depth else 0
        ref, Eb = G.head_block_ref(x, w9, bias, mode, a)
        carried = G._conv3x3(E, [abs(float(v)) for v in w9])
        if mode == 1:
            carried = carried + E.max(dim=1, keepdim=True)[0]
        x, E = ref, Eb + carried * (1 + 11 * U)  # Eb's 11 u |taps| term, taken on the engine's input: + 11 u carried
    ref, absum = _up(x)
    carried = _up(E)[0]
    absum = _up(x.abs() + E)[0]
    ref, Eo = G.bilinear_bound(ref, absum)
    return {"ref": ref, "bound": Eo + carried}


# ------------------------------------------------------------------------------------------------------------------
# tiers
# ------------------------------------------------------------------------------------------------------------------
def worst_ratio(got, st):
    """max |got - ref| / bound (> 1: outside)."""
    err = (got.to(F64) - st["ref"]).abs()
    return float((err / st["bound"]).nan_to_num(float("inf")).max())


def identical_fraction(got, st):
    """Tier B of an fp16 output: the fraction of elements (of those in b_mask, if any) bit-identical to rn16(ref_b)."""
    ref = st.get("ref_b", st["ref"])
    if "b_mask" in st:
        m = st["b_mask"]
        got, ref = got[m], ref[m]
    return G.bit_fraction(got, ref)


def rms_half_ulps(got, st):
    """Tier B of an fp32 output: RMS error / RMS half fp16 ulp of the output."""
    ref = st.get("ref_b", st["ref"])
    err = (got.to(F64) - ref).pow(2).mean().sqrt()
    return float(err / (ulp16(ref.abs()) / 2).pow(2).mean().sqrt())


def check(got, st, f16):
    """-> (report {worst, tier_b}, list of failure messages) of both tiers."""
    fails = []
    n, msg = G.violations(got, st["ref"], st["bound"])
    if n:
        fails.append("tier A: " + msg)
    if f16:
        tb, want = identical_fraction(got, st), st.get("b_min", FP16_IDENTICAL)
        if tb < want:
            fails.append(f"tier B: {tb:.4f} of the fp16 elements bit-identical to rn16(ref) < {want}")
    else:
        tb = rms_half_ulps(got, st)
        if not tb < FP32_RMS:
            fails.append(f"tier B: RMS error {tb:.3g} half fp16 ulps >= {FP32_RMS}")
    return {"worst": round(worst_ratio(got, st), 4), "tier_b": round(tb, 4)}, fails
