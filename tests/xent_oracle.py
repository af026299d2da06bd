"""float64 cross-entropy oracle for the device loss (csrc/xent.cuh) and the derived error bound of its fp32 sequence.

Oracle: CrossEntropyLoss(ignore_index) with mean reduction, in float64 over the given fp32 logits [B,K,H,W]: per
counted pixel logsumexp(v) - v_t, their mean; NaN when every pixel is ignored (0 / 0, as torch), and NaN for a target
outside [0, K) that is not ignore_index (the kernel's rule; torch asserts there).

Bound. The kernel computes, per pixel, in fp32 with u = 2^-24:
    m = max_k v_k                          (exact: comparisons)
    s = online sum of exp(v_k - m)         xent_lse_step: s <- fma(s, expf(m_old - v), 1) when v raises the maximum,
                                           s <- s + expf(v - m) otherwise
    l = fl(fl(m + logf(s)) - v_t)
Each term t_k = exp(v_k - m) of S = sum_k t_k (S >= 1: the maximal term is 1) reaches s through at most K expf factors
(its entry and each later rescale), each with an argument rounded once (fl(a - b), relative error <= u) and a result
within expf's 2 ulp <= 4u relative, and through at most K roundings of s (one per later fma or add, <= u each). The
argument differences of one term telescope to x_k = m - v_k >= 0, so their roundings move the term by at most
exp(u x_k); with c = (1 + 4u)^K (1 + u)^K:
    |s - S| <= S (c - 1) + c * sum_k t_k (exp(u x_k) - 1) + K 2^-125      (the last: expf results in the subnormal range)
and t_k (exp(u x_k) - 1) <= u x e^(-(1-u) x) <= u / ((1 - u) e), so with S >= 1
    rho = (c - 1) + c K u / ((1 - u) e) + K 2^-125     bounds |s / S - 1|.
Then |log s - log S| <= -log(1 - rho) =: e_s, logf adds <= 1 ulp <= 2u |log s|, and the two fp32 additions add
<= u |m + log s| and <= u |l|. Writing L = log S + e_s:
    |l - l_exact| <= e_s + 2u L + u (|m| + L)(1 + 2u) + u (|m| + L + |v_t|)(1 + 2u)^2
The mean of the counted pixels is within the mean of their bounds; the fp64 sum of N terms adds <= 2^-53 sum |l| to
the mean, and the final fp32 rounding u |mean|. The bound uses only K, u, the ulp bounds of expf / logf (CUDA C Programming
Guide, single-precision functions: 2 and 1 ulp, without fast-math) and the magnitudes of m, log S and v_t: derived,
not fitted.
"""
import math

import numpy as np

U = 2.0 ** -24
EXP_ULP = 2  # expf, max ulp error
LOG_ULP = 1  # logf, max ulp error


def _pixels(logits, target, ignore_index):
    """-> (counted mask [B,H,W], valid mask within it, m, log S, v_t) in float64 (v_t / m / log S at counted pixels)."""
    v = np.asarray(logits, dtype=np.float64)
    t = np.asarray(target, dtype=np.int64)
    K = v.shape[1]
    counted = t != ignore_index
    valid = counted & (t >= 0) & (t < K)
    m = v.max(axis=1)
    with np.errstate(invalid="ignore", over="ignore"):
        logS = np.log(np.exp(v - m[:, None]).sum(axis=1))
    vt = np.take_along_axis(v, np.where(valid, t, 0)[:, None], axis=1)[:, 0]
    return counted, valid, m, logS, vt


def xent_mean(logits, target, ignore_index=-1):
    """float64 mean cross-entropy of fp32 logits [B,K,H,W] against int target [B,H,W]."""
    counted, valid, m, logS, vt = _pixels(logits, target, ignore_index)
    loss = np.where(valid, m + logS - vt, np.nan)[counted]
    if loss.size == 0:
        return float("nan")
    return float(loss.mean())


def rho(K):
    """Relative error bound of the online sum s (module docstring)."""
    c = (1 + 2 * EXP_ULP * U) ** K * (1 + U) ** K
    return (c - 1) + c * K * U / ((1 - U) * math.e) + K * 2.0 ** -125


def pixel_bound(K, m, logS, vt):
    """Bound on |fp32 loss - exact loss| of one pixel, elementwise over arrays m, logS, vt (module docstring)."""
    r = rho(K)
    e_s = -math.log1p(-r)
    L = np.abs(logS) + e_s
    am = np.abs(m)
    return (e_s + 2 * LOG_ULP * U * L + U * (am + L) * (1 + 2 * U) +
            U * (am + L + np.abs(vt)) * (1 + 2 * U) ** 2)


def mean_bound(logits, target, ignore_index=-1):
    """Bound on |the device's fp32 mean loss - xent_mean| for these logits and targets (valid targets only)."""
    counted, valid, m, logS, vt = _pixels(logits, target, ignore_index)
    if not counted.any():
        return 0.0
    K = np.asarray(logits).shape[1]
    b = pixel_bound(K, m[counted], logS[counted], vt[counted])
    loss = np.abs(m + logS - vt)[counted] + b  # bounds |computed loss| per pixel
    # mean of the per-pixel bounds + the fp64 sum's (n - 1) 2^-53 sum |l| over n + the fp32 rounding of the mean
    return float(b.mean() + 2.0 ** -53 * loss.sum() + U * loss.mean())
