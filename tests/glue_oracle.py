"""Float64 references and error bounds for the glue kernels of the forward path (csrc/elementwise.cuh and
preprocess_kernel in csrc/evaluator.cuh).

Shared by tests/test_glue_gpu.py (against the kernels) and tests/test_glue_oracle_cpu.py (against float32 emulations of
each kernel's recipe, which must pass, and fake kernels with one planted defect each, which must fail). Plain torch:
CPU or CUDA tensors. u = 2^-24 is the fp32 unit roundoff; ulp16(a) / ulp32(a) are the spacings at magnitude a.

Bit-exact (no arithmetic, or one rounding that torch performs identically): patchify, readout_split, im2col_3x3_s2,
stem_im2col, maxpool3x3s2_nhwc, subsample2_nhwc, assemble_tokens (one fp32 add), the cls row of pos_resize,
channel_max, text_embed (__hadd of two rn16 values = torch's fp16 add) and text_eot_gather (first maximal id). Their
references are the torch one-liners in tests/test_glue_gpu.py.

layernorm (layernorm_kernel: one warp per row, lane-sequential sums of C/32 terms then 5 butterfly levels, so every
sum has depth n = C/32 + 5):

    m  = fl(sum x / C)             |m - mu| <= dmu = (n + 1) u sum|x| / C
    d  = fl(x - m)                 |d - (x - mu)| <= e = dmu (1 + u) + u |x - mu|
    ss = fl(sum d^2)               |ss - D| <= sum e (2|x - mu| + e) + (n + 1) u sum d^2,   D = sum (x - mu)^2
    v  = fl(fl(ss / C) + eps)      rel_v = |ss - D| / (D + C eps) + 2u
    r  = rsqrtf(v)                 2 ulp (CUDA programming guide) on top of the exact rsqrt: rel_r = rel_v / 2 / (1 - rel_v)
                                   + 2^-22
    y  = fl(fl(d r) g + b), rn16   (FMA or not: two roundings at most)

    |got - ref| <= |g| (e r + |x - mu| r rel_r + u |d r|) + u |g d r| + u |y| + ulp16(|y| + E) / 2

Bilinear kernels: the source coordinates and lambdas are formed in fp32 exactly as ATen forms them (bilinear_coords);
the blend is evaluated in float64 with those fp32 weights (hy = fp32(1 - ly), as ATen and the kernels round it). Every
kernel blends with at most two roundings per separable pass (a product and an add, or lerp2's FMA and product), so
|dy| <= 4u sum |w_i v_i| + O(u^2), written 5u to absorb the second-order terms. An `add` operand adds one rounding
(+ u |y|), an fp16 output adds half an fp16 ulp. For align_corners=False (pos_resize, preprocess) the coordinate is
`scale * (dst + 0.5) - 0.5`, which nvcc may contract into one FMA while ATen rounds the product: the coordinate then
moves by at most ulp32(src), and since the interpolant is continuous and piecewise linear in the coordinate (also
across a floor() boundary and the clamp at 0), the value moves by at most ulp32(src) * max |v_a - v_b| over the taps of
that axis. That slack is charged per axis by bilinear_ref(..., contract_slack=True).

head_block (head_block_kernel): up to 9 fmaf, + bias, + cmax, activation. acc error <= 11 u (sum|w x| + |bias| +
|cmax|); relu / leaky relu are 1-Lipschitz (leaky relu rounds 0.01 acc: + u |y|); tanhf is 1-Lipschitz with at most
2 ulp (CUDA programming guide): + 2 ulp32(|y|).

l2norm_f16 (norm rounded to fp16, then an fp16 division) and l2norm_scale (rn16(x / ||x||), then
rn16(logit_scale * that)): the only freedom is the fp32 summation order of ||x||^2, depth n = C/32 + 5, which moves the
norm by at most (n + 2) u relative. That is far below half an fp16 ulp, so l2norm_f16's fp16 norm is the float64 norm
rounded to fp16 or one of its neighbours: its bound is a one-ulp change of that fp16 norm. The contracts are the bound,
>= 99.9 % of the elements bit-identical to the float32 emulation (*_emulate), and exact bits where ||x||^2 is exact in
any order (rows of +-1 with C a power of two).
"""
import torch

U = 2.0 ** -24


def ulp32(a):
    a = torch.as_tensor(a, dtype=torch.float64).abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


def ulp16(a):
    a = torch.as_tensor(a, dtype=torch.float64).abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def r16(t):
    return t.to(torch.float16).to(torch.float64)


def violations(got, ref, bound):
    """(number of elements with |got - ref| > bound or non-finite got, description of the worst one)."""
    got = got.to(torch.float64)
    err = (got - ref).abs()
    bad = ~(err <= bound)
    n = int(bad.sum())
    if n == 0:
        return 0, "ok"
    excess = torch.where(bad, err - bound, torch.zeros_like(err)).nan_to_num(float("inf"))
    i = int(excess.flatten().argmax())
    return n, (f"{n} of {got.numel()} elements outside the bound; worst at flat index {i}: got "
               f"{got.flatten()[i].item():.9g}, ref {ref.flatten()[i].item():.9g}, bound {bound.flatten()[i].item():.3g}")


# ------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------
def layernorm_ref(x, gamma, beta, eps):
    """x [M, C] (fp32 or fp16 values) -> (float64 ref [M, C], bound [M, C]) for layernorm_kernel's fp16 output."""
    x = x.to(torch.float64)
    g = gamma.to(torch.float64)
    b = beta.to(torch.float64)
    C = x.shape[-1]
    n = C // 32 + 5
    mu = x.mean(-1, keepdim=True)
    xc = x - mu
    D = (xc * xc).sum(-1, keepdim=True)
    r = 1.0 / torch.sqrt(D / C + eps)
    ref = xc * r * g + b
    dmu = (n + 1) * U * x.abs().sum(-1, keepdim=True) / C
    e = dmu * (1 + U) + U * xc.abs()
    dss = (e * (2 * xc.abs() + e)).sum(-1, keepdim=True) + (n + 1) * U * ((xc.abs() + e) ** 2).sum(-1, keepdim=True)
    rel_v = dss / (D + C * eps) + 2 * U
    rel_r = rel_v / 2 / (1 - rel_v) + 2.0 ** -22
    dr = (xc.abs() + e) * r * (1 + rel_r)
    E = g.abs() * (e * r + xc.abs() * r * rel_r + U * dr) + U * g.abs() * dr + U * (ref.abs() + b.abs())
    return ref, E + ulp16(ref.abs() + E) / 2


def layernorm_emulate(x, gamma, beta, eps, *, ddof=0, use_eps=True):
    """float32 recipe of layernorm_kernel (torch's summation order), fp16 output. ddof / use_eps plant defects."""
    x = x.to(torch.float32)
    C = x.shape[-1]
    m = x.sum(-1, keepdim=True) / C
    d = x - m
    v = (d * d).sum(-1, keepdim=True) / (C - ddof)
    if use_eps:
        v = v + eps
    r = torch.rsqrt(v)
    return (d * r * gamma.float() + beta.float()).to(torch.float16)


# ------------------------------------------------------------------------------------------------------------------
# Bilinear interpolation
# ------------------------------------------------------------------------------------------------------------------
def bilinear_coords(n_in, n_out, align_corners, device="cpu"):
    """ATen's fp32 source taps for one axis: (i0, i1, w0, w1, src) with w1 = fp32 lambda, w0 = fp32(1 - lambda)."""
    dst = torch.arange(n_out, device=device, dtype=torch.float32)
    if align_corners:
        scale = torch.tensor(float(n_in - 1) / (n_out - 1) if n_out > 1 else 0.0, dtype=torch.float32)
        if n_out > 1:  # the fp32 quotient, rounded once
            scale = torch.tensor(float(n_in - 1), dtype=torch.float32) / torch.tensor(float(n_out - 1))
        src = scale.to(device) * dst
    else:
        scale = torch.tensor(float(n_in), dtype=torch.float32) / float(n_out)
        src = (scale.to(device) * (dst + 0.5) - 0.5).clamp_min(0.0)
    i0 = src.to(torch.int64).clamp_max(n_in - 1)
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    w1 = src - i0.to(torch.float32)
    w0 = 1.0 - w1
    return i0, i1, w0.double(), w1.double(), src.double()


def bilinear_ref(x, Ho, Wo, align_corners, *, contract_slack=False):
    """x [..., H, W] (any float dtype; values taken exactly) -> (float64 ref [..., Ho, Wo], sum |w_i v_i|, slack).
    slack: the FMA-contraction allowance of the coordinate expression (align_corners=False only), else 0."""
    x = x.to(torch.float64)
    H, W = x.shape[-2:]
    y0, y1, hy, ly, sy = bilinear_coords(H, Ho, align_corners, x.device)
    x0, x1, hx, lx, sx = bilinear_coords(W, Wo, align_corners, x.device)
    r0, r1 = x[..., y0, :], x[..., y1, :]
    v00, v01, v10, v11 = r0[..., x0], r0[..., x1], r1[..., x0], r1[..., x1]
    hy, ly = hy[:, None], ly[:, None]
    ref = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11)
    absum = hy * (hx * v00.abs() + lx * v01.abs()) + ly * (hx * v10.abs() + lx * v11.abs())
    slack = torch.zeros_like(ref)
    if contract_slack:
        dy = torch.maximum((v10 - v00).abs(), (v11 - v01).abs())
        dx = torch.maximum((v01 - v00).abs(), (v11 - v10).abs())
        slack = ulp32(sy)[:, None] * dy + ulp32(sx) * dx
    return ref, absum, slack


def bilinear_bound(ref, absum, slack=0.0, *, add=None, out_f16=False):
    """The bound of a bilinear kernel output (see the module docstring)."""
    E = 5 * U * absum + slack
    if add is not None:
        ref = ref + add.to(torch.float64)
        E = E + U * (ref.abs() + E)
    if out_f16:
        E = E + ulp16(ref.abs() + E) / 2
    return ref, E


def upsample2x_ref(x, *, add=None, out_f16=False):
    """bilinear x2, align_corners=True, of x [..., H, W] -> (ref, bound)."""
    H, W = x.shape[-2:]
    ref, absum, _ = bilinear_ref(x, 2 * H, 2 * W, True)
    return bilinear_bound(ref, absum, add=add, out_f16=out_f16)


def upsample2x_emulate(x, *, swap_x=False):
    """float32 recipe of the x2 align_corners=True kernels (vertical, then horizontal lerp). swap_x plants a defect."""
    x = x.to(torch.float32)
    H, W = x.shape[-2:]
    y0, y1, hy, ly, _ = bilinear_coords(H, 2 * H, True, x.device)
    x0, x1, hx, lx, _ = bilinear_coords(W, 2 * W, True, x.device)
    hy, ly, hx, lx = hy.float()[:, None], ly.float()[:, None], hx.float(), lx.float()
    if swap_x:
        hx, lx = lx, hx
    r0, r1 = x[..., y0, :], x[..., y1, :]
    return hy * (hx * r0[..., x0] + lx * r0[..., x1]) + ly * (hx * r1[..., x0] + lx * r1[..., x1])


# ------------------------------------------------------------------------------------------------------------------
# head_block
# ------------------------------------------------------------------------------------------------------------------
def _act64(t, act):
    if act == 1:
        return t.clamp_min(0)
    if act == 2:
        return torch.where(t > 0, t, 0.01 * t)
    if act == 3:
        return torch.tanh(t)
    return t


def _conv3x3(x, w9):
    """x [B, K, h, w] float64, shared 3x3 kernel, zero padding."""
    B, K, h, w = x.shape
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
    out = torch.zeros_like(x)
    for a in range(3):
        for b in range(3):
            out = out + w9[a * 3 + b] * xp[..., a:a + h, b:b + w]
    return out


def head_block_ref(x, w9, bias, mode, act):
    """x [B, K, h, w] -> (float64 ref, bound) of one head_block application (mode 1: + channel max)."""
    x = x.to(torch.float64)
    w9 = [float(torch.tensor(v, dtype=torch.float32)) for v in w9]
    bias = float(torch.tensor(bias, dtype=torch.float32))
    acc = _conv3x3(x, w9) + bias
    mag = _conv3x3(x.abs(), [abs(v) for v in w9]) + abs(bias)
    if mode == 1:
        cm = x.max(dim=1, keepdim=True)[0]
        acc = acc + cm
        mag = mag + cm.abs()
    E = 11 * U * mag
    ref = _act64(acc, act)
    if act == 2:
        E = E + U * ref.abs()
    elif act == 3:
        E = E + 2 * ulp32(ref.abs() + E)
    return ref, E + 1e-45


def head_block_emulate(x, w9, bias, mode, act, *, act_before_cmax=False):
    """float32 recipe of head_block_kernel. act_before_cmax plants a defect."""
    x = x.to(torch.float32)
    B, K, h, w = x.shape
    wt = torch.tensor(w9, dtype=torch.float32, device=x.device).view(1, 1, 3, 3)
    acc = torch.nn.functional.conv2d(x.reshape(B * K, 1, h, w), wt, padding=1).view(B, K, h, w) + bias
    f = {0: lambda t: t, 1: torch.relu, 2: lambda t: torch.nn.functional.leaky_relu(t, 0.01), 3: torch.tanh}[act]
    if mode == 1:
        cm = x.max(dim=1, keepdim=True)[0]
        return f(acc) + cm if act_before_cmax else f(acc + cm)
    return f(acc)


# ------------------------------------------------------------------------------------------------------------------
# L2 norms
# ------------------------------------------------------------------------------------------------------------------
def _step16(h, up):
    bits = h.view(torch.int16).to(torch.int32)
    bits = bits + (1 if up else -1)  # positive values only: the integer order of fp16 bits is their value order
    return bits.to(torch.int16).view(torch.float16)


def l2norm_f16_ref(x):
    """x fp16 [M, C] -> (float64 ref = x / rn16(||x||), bound): the fp16 norm may be off by one fp16 ulp."""
    x64 = x.to(torch.float64)
    n16 = r16(x64.norm(dim=-1, keepdim=True))
    lo = _step16(n16.to(torch.float16), False).to(torch.float64)
    hi = _step16(n16.to(torch.float16), True).to(torch.float64)
    ref = x64 / n16
    dev = torch.maximum(x64.abs() / lo - ref.abs(), ref.abs() - x64.abs() / hi)
    qmax = x64.abs() / lo
    return ref, dev + U * qmax + ulp16(qmax) / 2


def l2norm_f16_emulate(x, *, round_norm=True):
    """float32 recipe of l2norm_f16_kernel. round_norm=False plants a defect (the norm stays fp32)."""
    f = x.to(torch.float32)
    nrm = torch.sqrt((f * f).sum(-1, keepdim=True))
    if round_norm:
        nrm = nrm.half().float()
    return (f / nrm).half()


def l2norm_scale_ref(x, logit_scale):
    """x fp32 [M, C] -> (float64 ref = ls * x / ||x||, bound)."""
    x64 = x.to(torch.float64)
    C = x.shape[-1]
    ls = float(torch.tensor(logit_scale, dtype=torch.float32))
    delta = (C // 32 + 7) * U
    q = x64 / x64.norm(dim=-1, keepdim=True)
    qa = q.abs() * (1 + delta)
    e1 = delta * q.abs() + ulp16(qa) / 2  # rn16(x / fp32 norm), fp32 division included in delta
    y = ls * (qa + ulp16(qa) / 2)
    E = ls * e1 + U * y + ulp16(y) / 2
    return ls * q, E


def l2norm_scale_emulate(x, logit_scale, *, scale_first=False):
    """float32 recipe of l2norm_scale_kernel. scale_first plants a defect (logit_scale applied before the fp16 rounding)."""
    f = x.to(torch.float32)
    nrm = torch.sqrt((f * f).sum(-1, keepdim=True))
    ls = torch.tensor(logit_scale, dtype=torch.float32, device=f.device)
    if scale_first:
        return (ls * (f / nrm)).half()
    return (ls * (f / nrm).half().float()).half()


def bit_fraction(got, want):
    """Fraction of elements whose fp16 bits agree."""
    return (got.to(torch.float16).view(torch.int16) == want.to(torch.float16).view(torch.int16)).double().mean().item()
