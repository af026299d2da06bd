"""Shared helpers for the model-level parity tests (CUDA path vs. the CPU oracle)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import lseg_oracle as O  # noqa: E402
from oracle import synth  # noqa: E402

NET_KW = dict(backbone="clip_vitl16_384", features=256, crop_size=480, arch_option=0, block_depth=0,
              activation="lrelu")  # kwargs of modules/lseg_module.py:76-84

_STATE = {}


def state_dict(seed=0, backbone="clip_vitl16_384"):
    key = seed if backbone == "clip_vitl16_384" else (seed, backbone)
    if key not in _STATE:
        _STATE[key] = synth.make_state_dict(seed, backbone=backbone)
    return _STATE[key]


def rel_err(got, ref):
    """max |got-ref| / max |ref| (the '1e-3 relative' metric of BASELINE.json's north_star)."""
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-12)).item()


def on_lattice(t, lat):
    """t [B, K, H, W] sampled on the regular pixel lattice a golden fixture stores (lat [B, K, H / s, W / s])."""
    s = t.shape[-1] // lat.shape[-1]
    return t[:, :, ::s, ::s]


def rms_rel_err(got, ref):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    return ((got - ref).pow(2).mean().sqrt() / (ref.pow(2).mean().sqrt() + 1e-12)).item()


def argmax_report(got, ref, margin_eps):
    """Mask agreement + the margin rule: every mismatching pixel must be a near-tie in the ORACLE
    (top-2 logit margin < margin_eps) — see SURVEY.md section 7 'hard parts'."""
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    ga, ra = got.argmax(1), ref.argmax(1)
    mism = ga != ra
    if ref.shape[1] > 1:
        top2 = ref.topk(2, dim=1).values
        margin = top2[:, 0] - top2[:, 1]
    else:
        margin = torch.full(ra.shape, float("inf"))
    n_mis = int(mism.sum())
    worst = float(margin[mism].max()) if n_mis else 0.0
    return {
        "pixels": int(mism.numel()),
        "mismatch": n_mis,
        "agree_frac": 1.0 - n_mis / mism.numel(),
        "worst_mismatch_margin": worst,
        "near_tie_frac": float((margin < margin_eps).float().mean()),
        "ok": bool(n_mis == 0 or worst < margin_eps),
    }


def argmax_report_from_mask(mask, ref, margin_eps):
    """Same rule for a class mask (int64 [B,H,W]) instead of logits."""
    ref = ref.detach().float().cpu()
    mask = mask.detach().cpu()
    ra = ref.argmax(1)
    mism = mask != ra
    top2 = ref.topk(2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    n_mis = int(mism.sum())
    worst = float(margin[mism].max()) if n_mis else 0.0
    return {"pixels": int(mism.numel()), "mismatch": n_mis, "agree_frac": 1.0 - n_mis / mism.numel(),
            "worst_mismatch_margin": worst, "ok": bool(n_mis == 0 or worst < margin_eps)}


def oracle_forward(x, tokens, seed=0, stages=True):
    oracle_threads()
    return O.lseg_forward(x, tokens, state_dict(seed), return_stages=stages)


def oracle_threads():
    """torch's CPU kernels on these small matrices get SLOWER beyond ~16 threads (measured 64 s per 480x480
    forward with 128 threads vs 1.5 s with 16 on the GPU box's host), and GPU-box time is budgeted."""
    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))
