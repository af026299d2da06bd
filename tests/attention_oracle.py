"""Float64 references, error bounds and a rounding-point emulation for the two attention kernels.

Shared by tests/test_attention_gpu.py (against the kernels) and tests/test_attention_oracle_cpu.py (against fake
kernels, to show the bounds catch a dropped key or a wrong causal diagonal). Plain torch: CPU or CUDA tensors.

mhsa_oracle bounds csrc/mhsa.cuh, which computes per query row, over 64-key tiles j (the derivation):

    S_j = q.k_j in fp32 on the tensor cores              64 products (exact) summed: |dS_j| <= 64 u_tc sum_k |q_k k_jk|
    x_j = fmaf(S_j, c, -mu), c = fp32(0.125 log2 e)     |dx_j| <= c |S_j| u + |x_j| u, and |x_j| <= R, the row's score
                                                          range in log2 units (mu is the running maximum, so x_j <= 0)
    p_j = ex2(x_j)                                       relative eps_exp: 2 ulp = 2^-22 for ex2.approx.ftz (MUFU,
                                                          NVIDIA's documented bound for the instruction behind exp2f);
                                                          7.5e-5 for exp2_poly<3> (tools/fit_exp2.py) in the POLY
                                                          instantiations. The -126 clamp of the POLY path only moves
                                                          p_j < 2^-126, which rounds to fp16 zero either way.
    rescale when the running max moves: O *= f, l = l f + sum, f = ex2(m_old - mu_new)
                                                          per rescale: eps_ex2 on f, u R on the subtraction, u on O
    P_j = fp16(p_j)                                      relative 2^-11, or absolute 2^-25 where P_j is subnormal
    O  += P V on the tensor cores                        n_vis additions (masked keys add exact zeros)
    l   = sum of the fp32 p_j (not of P_j)               per thread 16 keys per tile, l f + sum per tile, 2 shuffles
    out = fp16(O * (1 / l))                              2 roundings, then one fp16 rounding

An error in p_j that reaches both O and l (S, exponent, rescale: relative e_j <= eps_w) moves the output by
sum_j w_j (e_j - e_mean) v_jd / (1 + e_mean), at most 2 eps_w / (1 - eps_w) * sum_j w_j |v_jd|. The fp16 rounding of P
reaches only O. With w the float64 softmax weights, p_j = exp(s_j - max s) and n_kt the row's key-tile count:

    |got - ref| <= eps_tot * sum_j w_j |v_jd|  +  2^-25 (1 + eps_tot) * sum_j |v_jd| / sum_j p_j  +  ulp16(|ref|)

    eps_w   = (1 + eps_exp) (1 + 2^-22)^n_kt * exp(0.125 (64 u_tc A + u max_j |S_j|) + ln2 u R (1 + n_kt)) - 1
    eps_tot = (1 + 2^-11) (1 + 2 eps_w / (1 - eps_w)) (1 + n_vis u_tc + (3 n_kt + 13) u) - 1

with A = max_j sum_k |q_k k_jk|, u = 2^-24 (fp32, round to nearest) and u_tc = 2^-23: tensor-core fp32 accumulation is
not specified as round-to-nearest, so it is charged one full ulp per addition. Against the plain form
eps_p = 2^-11 + eps_exp + N 2^-24 + 0.125 * 64 * 2^-24 * A, this charges the tensor-core sums twice, counts the rescales
(each one a MUFU exponential and a rounding), and doubles the terms that move p_j in both O and l (the
renormalisation term above). All of those are rounding points of the kernel, not slack.
"""
import math

import torch

# (B, N, heads, causal, amp): the shapes tests/test_ops_gpu.py::test_mhsa runs every variant on;
# tests/test_attention_gpu.py runs them through every input family
MHSA_SHAPES = [
    (2, 901, 16, False, 1.0), (3, 77, 8, True, 1.0), (1, 37, 16, False, 1.0), (1, 300, 2, True, 1.0),
    # key-tile boundary cases of the wgmma flash-attention kernel (64 keys per K/V tile): a single tile, exact multiples,
    # 1..2 keys in the tail tile, odd/even tile counts; amp 3 makes the running-max offset move (O rescale path)
    (1, 64, 1, False, 1.0), (1, 65, 1, True, 1.0), (1, 128, 2, False, 1.0), (1, 130, 2, False, 3.0),
    (1, 1025, 2, False, 1.0), (2, 300, 2, False, 3.0), (1, 193, 1, True, 3.0),
    # token counts of BASELINE.json configs[4]: 704^2 -> 1937, 736^2 -> 2117 (34 key tiles; 17 query tiles)
    (1, 1937, 4, False, 1.0), (1, 2117, 3, False, 1.0), (1, 2117, 1, False, 3.0)]

LOG2E = 1.4426950408889634
U = 2.0 ** -24       # fp32 unit roundoff, round to nearest
U_TC = 2.0 ** -23    # one fp32 ulp per tensor-core accumulation step
EPS_EX2 = 2.0 ** -22
EPS_POLY = 7.5e-5
EPS_P16 = 2.0 ** -11
SUBNORMAL_P = 2.0 ** -25


def ulp16(a):
    """fp16 ulp at |a| (float64 tensor), 2^-24 in the subnormal range."""
    e = torch.floor(torch.log2(a.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def _row_counts(N, causal, device):
    r = torch.arange(N, device=device, dtype=torch.float64)
    if not causal:
        return torch.full_like(r, float(N)), torch.full_like(r, float(math.ceil(N / 64)))
    kv_end = torch.clamp((torch.div(r, 128, rounding_mode="floor") + 1) * 128, max=N)
    return r + 1, torch.ceil(kv_end / 64)


def mhsa_oracle(qkv, B, N, heads, causal, eps_exp=EPS_EX2, drop_key=None, diag=True):
    """(ref, bound), float64 [B*N, heads*64], for qkv fp16 [B, N, 3*heads*64]. drop_key / diag=False build the
    reference of a wrong kernel (CPU rehearsal only)."""
    D = heads * 64
    x = qkv.reshape(B, N, 3, heads, 64)
    ref = torch.empty((B, N, heads, 64), dtype=torch.float64, device=qkv.device)
    bound = torch.empty_like(ref)
    n_vis, n_kt = _row_counts(N, causal, qkv.device)
    n_vis, n_kt = n_vis.view(1, N, 1), n_kt.view(1, N, 1)  # per query row
    vis = torch.ones((N, N), dtype=torch.bool, device=qkv.device)
    if causal:
        vis = torch.tril(vis, 0 if diag else -1)
    if drop_key is not None:
        vis[:, drop_key] = False
    hc = max(1, min(heads, (1 << 25) // (N * N)))  # heads per chunk: <= 32M float64 scores at a time
    for b in range(B):
        for h0 in range(0, heads, hc):
            h1 = min(heads, h0 + hc)
            q, k, v = (x[b, :, i, h0:h1].transpose(0, 1).double() for i in range(3))  # [hc, N, 64]
            S = q @ k.transpose(1, 2)
            Sm = S.masked_fill(~vis, float("-inf"))
            smax = Sm.amax(-1, keepdim=True)
            p = torch.exp(0.125 * (Sm - smax))
            P = p.sum(-1, keepdim=True)
            w = p / P
            ref[b, :, h0:h1] = (w @ v).transpose(0, 1)
            av = v.abs()
            wv = w @ av
            sv = vis.double() @ av
            A = (q.abs() @ k.abs().transpose(1, 2)).masked_fill(~vis, 0).amax(-1, keepdim=True)
            s_abs = S.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
            smin = S.masked_fill(~vis, float("inf")).amin(-1, keepdim=True)
            R = 0.125 * LOG2E * (smax - smin).nan_to_num(0.0)
            dlog = 0.125 * (64 * U_TC * A + U * s_abs) + math.log(2) * U * R * (1 + n_kt)
            eps_w = (1 + eps_exp) * (1 + EPS_EX2) ** n_kt * torch.exp(dlog) - 1
            eps_tot = (1 + EPS_P16) * (1 + 2 * eps_w / (1 - eps_w)) * (1 + n_vis * U_TC + (3 * n_kt + 13) * U) - 1
            bnd = eps_tot * wv + SUBNORMAL_P * (1 + eps_tot) * sv / P
            bound[b, :, h0:h1] = bnd.transpose(0, 1)
    ref = ref.reshape(B * N, D)
    bound = bound.reshape(B * N, D) + ulp16(ref)
    return ref, bound


def flat_reference(v, causal):
    """q = 0: every visible key weighs the same. v: [B, N, heads, 64] -> float64 [B*N, heads*64]."""
    B, N = v.shape[:2]
    vd = v.double()
    if causal:
        ref = vd.cumsum(1) / torch.arange(1, N + 1, device=v.device, dtype=torch.float64).view(1, N, 1, 1)
    else:
        ref = vd.mean(1, keepdim=True).expand_as(vd)
    return ref.reshape(B * N, -1)


def flat_tolerance(ref, eps_exp):
    """P = fp16(ex2(0)) = 1 exactly, PV and l are integer sums; l is off by at most eps_exp relative (POLY), 1 / l and
    O / l round once each in fp32, the store rounds to fp16."""
    return 0.5 * ulp16(ref) + (2.0 ** -22 + eps_exp) * ref.abs()


def violations(got, ref, bound):
    """(count, message about the worst element) of |got - ref| > bound; NaN / inf in got always counts."""
    g = got.double()
    diff = (g - ref).abs()
    bad = ~(diff <= bound)
    n = int(bad.sum())
    if n == 0:
        return 0, ""
    ratio = torch.where(bad, (diff / bound).nan_to_num(float("inf")), torch.zeros_like(diff))
    i = int(ratio.reshape(-1).argmax())
    r, c = divmod(i, ref.shape[-1])
    return n, (f"{n} of {ref.numel()} elements outside the bound; worst at row {r} col {c}: got {g[r, c].item():.7g}, "
               f"want {ref[r, c].item():.7g}, |diff| {diff[r, c].item():.3g} > bound {bound[r, c].item():.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# lseg_text_attn: the kernel's rounding points, in the kernel's order, in float32
# ---------------------------------------------------------------------------------------------------------------------
def text_attn_emulate(qkv, K, L, heads, drop_last_pv=False):
    """fp16 [K*L, heads*64] as csrc/text_attn.cuh computes it:
      q8 = fp16(q * 0.125);  S_ij = fp16(fmaf chain over d = 0..63 of q8_id k_jd)  (fp16 x fp16 products are exact in
      fp32, so each step is one rounded fp32 add);  e_j = expf(S_ij - max_j S_ij);  lane l of the row's warp sums
      e_l, e_l+32, e_l+64 in that order, then the xor-16, 8, 4, 2, 1 butterfly;  P_ij = fp16(e_j / sum);
      out_i = fp16(fmaf chain over j = 0..i of P_ij v_j).
    Only expf can differ from the kernel (torch's exp against the kernel's expf). drop_last_pv: the PV chain stops at
    j < i (CPU rehearsal of a wrong kernel)."""
    D = heads * 64
    x = qkv.reshape(K, L, 3, heads, 64).permute(2, 0, 3, 1, 4)  # [3, K, heads, L, 64]
    q8 = (x[0] * 0.125).float()  # an fp16 product, rounded to fp16 as __hmul2 does
    k, v = x[1].float(), x[2].float()
    acc = torch.zeros((K, heads, L, L), dtype=torch.float32, device=qkv.device)
    for d in range(64):
        acc = acc + q8[..., :, None, d] * k[..., None, :, d]
    s = acc.half().float()
    vis = torch.ones((L, L), dtype=torch.bool, device=qkv.device).tril()
    s = s.masked_fill(~vis, float("-inf"))
    mx = s.amax(-1, keepdim=True)
    e = torch.exp(s - mx).masked_fill(~vis, 0.0)
    e96 = torch.zeros((K, heads, L, 96), dtype=torch.float32, device=qkv.device)
    e96[..., :L] = e
    lanes = torch.zeros((K, heads, L, 32), dtype=torch.float32, device=qkv.device)
    for t in range(3):
        lanes = lanes + e96[..., 32 * t:32 * t + 32]
    idx = torch.arange(32, device=qkv.device)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[..., idx ^ o]
    tot = lanes[..., :1]
    p = (e / tot).half().float().masked_fill(~vis, 0.0)
    if drop_last_pv:
        p = p.masked_fill(torch.eye(L, dtype=torch.bool, device=qkv.device), 0.0)
    o = torch.zeros((K, heads, L, 64), dtype=torch.float32, device=qkv.device)
    for j in range(L):
        o = o + p[..., :, j, None] * v[..., j, None, :]
    return o.half().permute(0, 2, 1, 3).reshape(K * L, D)


def text_attn_flat(v, K, L, heads):
    """q = 0: P_ij = fp16(1 / (i + 1)) for j <= i, and out_i = fp16(sum in order of P_ij v_j). v fp16 [K, L, heads, 64]."""
    pr = (1.0 / torch.arange(1, L + 1, device=v.device, dtype=torch.float32)).half().float()  # [L]
    vf = v.float().permute(0, 2, 1, 3)  # [K, heads, L, 64]
    rows = torch.arange(L, device=v.device).view(1, 1, L, 1)
    o = torch.zeros_like(vf)
    for j in range(L):  # rows i >= j add P_i v_j (an exact product); rows i < j add an exact zero
        o = o + pr.view(1, 1, L, 1) * vf[:, :, j:j + 1] * (rows >= j)
    return o.half().permute(0, 2, 1, 3).reshape(K * L, heads * 64)
