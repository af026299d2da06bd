"""The attention oracles of tests/attention_oracle.py have teeth: on CPU, a "kernel" that is the float64 reference
rounded to fp16 passes the mhsa bound and the exact key-count check, while the same with one key dropped or with the
causal diagonal excluded fails them; the text-attention emulation matches its closed form at q = 0 and tells a PV chain
that stops one key early from the right one."""
import pytest
import torch

from attention_oracle import (EPS_EX2, EPS_POLY, flat_reference, flat_tolerance, mhsa_oracle, text_attn_emulate,
                              text_attn_flat, violations)


def _flat_qkv(B, N, heads, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, N, 3, heads, 64), generator=g)
    x[:, :, 0] = 0
    x[:, :, 2] = torch.randint(-4, 5, (B, N, heads, 64), generator=g).float()
    return x.half().reshape(B, N, 3 * heads * 64)


def _random_qkv(B, N, heads, seed, amp=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B, N, 3 * heads * 64), generator=g) * amp).half()


@pytest.mark.parametrize("N,causal", [(130, False), (130, True), (64, True), (193, False)])
@pytest.mark.parametrize("eps_exp", [EPS_EX2, EPS_POLY])
def test_rounded_reference_passes_and_wrong_keys_fail(N, causal, eps_exp):
    B, heads = 2, 2
    qkv = _flat_qkv(B, N, heads, 5)
    ref, bound = mhsa_oracle(qkv, B, N, heads, causal, eps_exp)
    flat = flat_reference(qkv.view(B, N, 3, heads, 64)[:, :, 2], causal)
    tol = flat_tolerance(flat, eps_exp)
    good = ref.half()
    assert violations(good, ref, bound)[0] == 0
    assert violations(good, flat, tol)[0] == 0
    for drop in (0, 63, N - 1):
        wrong = mhsa_oracle(qkv, B, N, heads, causal, eps_exp, drop_key=drop)[0].half()
        assert violations(wrong, ref, bound)[0] > 0, f"dropping key {drop} passes the bound"
        assert violations(wrong, flat, tol)[0] > 0, f"dropping key {drop} passes the key-count check"
    if causal:
        wrong = mhsa_oracle(qkv, B, N, heads, causal, eps_exp, diag=False)[0].half()
        assert violations(wrong, ref, bound)[0] > 0, "excluding the causal diagonal passes the bound"
        assert violations(wrong, flat, tol)[0] > 0, "excluding the causal diagonal passes the key-count check"
    # random scores: the rounded reference passes; a dropped key fails
    qkv = _random_qkv(B, N, heads, 6, 3.0)
    ref, bound = mhsa_oracle(qkv, B, N, heads, causal, eps_exp)
    assert violations(ref.half(), ref, bound)[0] == 0
    wrong = mhsa_oracle(qkv, B, N, heads, causal, eps_exp, drop_key=N // 2)[0].half()
    assert violations(wrong, ref, bound)[0] > 0


def test_bound_is_tight_where_it_matters():
    """With random scores most of the bound is the fp16 rounding of P: 2^-11 of sum_j w_j |v_j| plus an ulp of the
    result, not a multiple of it."""
    B, N, heads = 1, 2117, 1
    qkv = _random_qkv(B, N, heads, 7)
    ref, bound = mhsa_oracle(qkv, B, N, heads, False)
    x = qkv.view(B, N, 3, heads, 64).double()
    s = (x[0, :, 0, 0] @ x[0, :, 1, 0].t()) * 0.125
    wv = s.softmax(-1) @ x[0, :, 2, 0].abs()
    assert float((bound / (wv * 2.0 ** -11)).median()) < 3.0


@pytest.mark.parametrize("K,L,heads", [(2, 1, 8), (3, 33, 8), (2, 77, 12)])
def test_text_emulation(K, L, heads):
    g = torch.Generator().manual_seed(9)
    qkv = (torch.randn((K, L, 3 * heads * 64), generator=g) * 1.5).half()
    flat = qkv.clone().view(K, L, 3, heads, 64)
    flat[:, :, 0] = 0
    v = flat[:, :, 2]
    flat = flat.view(K, L, 3 * heads * 64)
    emu = text_attn_emulate(flat, K, L, heads)
    assert torch.equal(emu.view(torch.int16), text_attn_flat(v, K, L, heads).view(torch.int16))
    if L > 1:
        short = text_attn_emulate(flat, K, L, heads, drop_last_pv=True)
        assert not torch.equal(short.view(torch.int16), emu.view(torch.int16))
