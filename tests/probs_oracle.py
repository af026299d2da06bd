"""Float64 reference and error bound of the attention-probability kernel (csrc/attn_probs.cuh), beside the MHSA ones of
tests/attention_oracle.py (same constants, same conventions). Plain torch: CPU or CUDA tensors.

The kernel computes, per query row i and key j, over n_kt 64-key tiles (the derivation):

    S_ij = q_i.k_j in fp32 on the tensor cores          64 exact products summed: |dS_ij| <= 64 u_tc A_ij,
                                                          A_ij = sum_d |q_id k_jd|
    c = fp32(0.125 log2 e)                               relative u
    pass 1, per tile t: m_t = max(m_{t-1}, fp32(max_j S_ij * c)) (a running offset: it cancels between numerator and
        denominator as long as every term is taken against the same final m, which the rescales below carry)
        e_ij = ex2(fmaf(S_ij, c, -m_t))                  fmaf: |dx| <= c |S_ij| u + |x_ij| u with |x_ij| <= R_i (the row's
                                                          score range in log2 units); ex2.approx.ftz relative eps_ex2
        l = l * f + sum_tile e, f = ex2(m_{t-1} - m_t)   per rescale: eps_ex2 on f, u R_i on the subtraction
    pass 2: p_ij = ex2(fmaf(S_ij, c, -m_final)) * fp32(1 / l)
                                                          the same fmaf / ex2 error as in pass 1 on the numerator, then
                                                          the reciprocal and the product: 2 roundings

Write w_ij for the float64 softmax of 0.125 q_i.k_j. Every numerator and every term of l carries a relative error of at
most eps_w (its exponent is off by at most dlog_i, plus at most n_kt + 1 ex2 errors along its rescale chain):

    eps_w_i = (1 + eps_ex2)^(n_kt + 1) exp(0.125 (64 u_tc A_i + u S_i) + ln2 u R_i (n_kt + 2)) - 1

with A_i = max_j A_ij and S_i = max_j |S_ij|. l is a sum of positive terms: each thread adds its 16 terms of a tile in
order, then l f + sum and, at the end, two shuffle additions, so no term passes more than 2 n_kt + 20 fp32 roundings
(the charge of one unit roundoff each). The ratio numerator / l then has relative error

    eps_tot_i = (1 + eps_w_i) / (1 - eps_w_i) * (1 + u)^(2 n_kt + 22) - 1      (the 22 includes 1 / l and the product)

ex2.approx.ftz flushes results below 2^-126 to zero, and l >= 1 (the row's maximal key contributes ex2(~0) = 1), so a
term that underflows moves p by less than 2^-126. The bound per element:

    |p_ij - w_ij| <= eps_tot_i * w_ij + 2^-125

and per row, |sum_j p_ij - 1| <= sum_j (bound_ij) + N 2^-52 (the float64 row sum of the reference).

With q = 0 (the `flat` family) every S is exactly 0, m = 0, e = ex2(0) = 1 exactly, l = N exactly (integers below 2^24)
and p = fp32(1 / N) in every element, which flat_probs states exactly.
"""
import math

import torch

from attention_oracle import EPS_EX2, LOG2E, U, U_TC

UNDERFLOW = 2.0 ** -125


def probs_oracle(q, k):
    """(w, bound), float64 [..., N, N], for fp16 (or fp16-valued) q, k [..., N, 64] of one or more (image, head) planes:
    w = softmax(0.125 q k^T) and the kernel's derived per-element bound |p - w| <= bound."""
    qd, kd = q.double(), k.double()
    N = q.shape[-2]
    n_kt = math.ceil(N / 64)
    S = qd @ kd.transpose(-1, -2)
    smax = S.amax(-1, keepdim=True)
    p = torch.exp(0.125 * (S - smax))
    w = p / p.sum(-1, keepdim=True)
    A = (qd.abs() @ kd.abs().transpose(-1, -2)).amax(-1, keepdim=True)
    s_abs = S.abs().amax(-1, keepdim=True)
    R = 0.125 * LOG2E * (smax - S.amin(-1, keepdim=True))
    dlog = 0.125 * (64 * U_TC * A + U * s_abs) + math.log(2) * U * R * (n_kt + 2)
    eps_w = (1 + EPS_EX2) ** (n_kt + 1) * torch.exp(dlog) - 1
    eps_tot = (1 + eps_w) / (1 - eps_w) * (1 + U) ** (2 * n_kt + 22) - 1
    return w, eps_tot * w + UNDERFLOW


def row_sum_bound(bound):
    """|sum_j p_ij - 1| bound per row from the element bounds (float64 [..., N, N] -> [..., N])."""
    N = bound.shape[-1]
    return bound.sum(-1) + N * 2.0 ** -52


def flat_probs(N):
    """q = 0: every element is exactly fp32(1 / N) (an fp32 tensor holding that value)."""
    return torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(N), dtype=torch.float32)


def violations(got, ref, bound):
    """(count, message about the worst element) of |got - ref| > bound over [..., N, N]; NaN / inf always counts."""
    diff = (got.double() - ref).abs()
    bad = ~(diff <= bound)
    n = int(bad.sum())
    if n == 0:
        return 0, ""
    ratio = torch.where(bad, (diff / bound).nan_to_num(float("inf")), torch.zeros_like(diff))
    i = int(ratio.reshape(-1).argmax())
    idx = []
    for s in reversed(ref.shape):
        i, r = divmod(i, s)
        idx.append(r)
    idx = tuple(reversed(idx))
    return n, (f"{n} of {ref.numel()} elements outside the bound; worst at {idx}: got {got[idx].item():.9g}, "
               f"want {ref[idx].item():.9g}, |diff| {diff[idx].item():.3g} > bound {bound[idx].item():.3g}")
