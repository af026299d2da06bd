"""CPU: the recorded attention maps (enable_attention_hooks) of the oracle against the unmodified reference
(tests/golden/ref_attention.npz, oracle/make_golden_attention.py), and lseg_net.get_mean_attention_map against the
reference's own function on those tensors.

Tolerance of the oracle against the fixture, derived: both run the same torch ops in the same order, so they can differ
only where this machine's CPU kernels sum an fp32 GEMM in another order than the machine that wrote the fixture. Such a
reordering moves every fp32 activation of the trunk by a few ulps; RHO = 2^-16 charges q and k of the hooked block
(after up to 24 blocks) 2^-16 relative to their plane's largest magnitude — 256 ulps. A score moves by at most
delta_i = 0.125 * RHO * (Qmax ||k_j||_1 + Kmax ||q_i||_1) in row i, and a softmax row whose scores move by at most delta
moves each probability by at most w (exp(2 delta) - 1), plus 2^-24 for the fp32 rounding of the value itself.
"""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import vit_attention_oracle as A
from parity_util import O, state_dict, synth

GOLD = os.path.join(os.path.dirname(__file__), "golden")
torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
RHO = 2.0 ** -16
CASES = [("small", 2, 64, 96, 2064), ("s480", 1, 480, 480, 1480)]


def _fixture():
    return np.load(os.path.join(GOLD, "ref_attention.npz"))


def _tolerance(q, k, w):
    """Element bound |oracle - fixture| for q, k [B, heads, N, 64] and the probabilities w [B, heads, rows, N]."""
    qmax = q.abs().amax(dim=(-2, -1)).unsqueeze(-1)  # [B, heads, 1]
    kmax = k.abs().amax(dim=(-2, -1)).unsqueeze(-1)
    k1 = k.abs().sum(-1).amax(-1, keepdim=True)  # max_j ||k_j||_1, [B, heads, 1]
    q1 = q.abs().sum(-1)                          # ||q_i||_1, [B, heads, N]
    delta = 0.125 * RHO * (qmax * k1 + kmax * q1)  # [B, heads, N] per query row
    return w.abs() * torch.expm1(2 * delta.unsqueeze(-1)) + 2.0 ** -24


@pytest.mark.parametrize("tag,B,H,W,seed", CASES)
def test_oracle_attention_matches_reference(tag, B, H, W, seed):
    z = _fixture()
    x = synth.make_image(B, H, W, seed=seed)
    qk, taps = {}, []
    got = A.vit_attention_maps(x, state_dict(0), taps_out=taps, qk_out=qk)
    assert sorted(got) == ["attn_1", "attn_2", "attn_3", "attn_4"]
    N = (H // 16) * (W // 16) + 1
    rows = list(range(N)) if tag == "small" else [int(r) for r in z["s480_rows"]]
    for name, a in got.items():
        assert a.shape == (B, 16, N, N) and a.dtype == torch.float32
        ref = torch.from_numpy(z[f"{tag}_{name}"])
        sel = a[:, :, rows]
        assert sel.shape == ref.shape
        q, k = qk[name]
        tol = _tolerance(q, k, a)[:, :, rows]
        err = (sel - ref).abs()
        assert bool((err <= tol).all()), (name, (err - tol).max().item())
    if tag == "small":  # the trunk is the oracle's own: the same taps, bit for bit
        ref_taps = O.vit_forward_flex(x, state_dict(0))
        for t, r in zip(taps, ref_taps):
            assert torch.equal(t, r)


def test_mean_attention_map_matches_reference():
    """get_mean_attention_map on the fixture's reference tensors equals the reference function's output exactly: the
    same torch ops in the same order. B = 1 averages over the heads ([H, W]); B = 2 over the images ([heads, H, W])."""
    lseg_net = importlib.import_module("lang-seg_b200.lseg_net")
    z = _fixture()
    s2 = int(z["mean_b2_stride"])
    n = 0
    for name in ("attn_1", "attn_4"):
        attn = torch.from_numpy(z[f"small_{name}"])
        for t in (int(v) for v in z["mean_tokens"]):
            m1 = lseg_net.get_mean_attention_map(attn[:1], t, (1, 3, 64, 96))
            assert m1.shape == (64, 96)
            assert torch.equal(m1, torch.from_numpy(z[f"mean_b1_t{t}_{name}"]))
            m2 = lseg_net.get_mean_attention_map(attn, t, (2, 3, 64, 96))
            assert m2.shape == (16, 64, 96)
            assert torch.equal(m2[:, ::s2, ::s2], torch.from_numpy(z[f"mean_b2_t{t}_{name}"]))
            n += 2
    assert n == 8
