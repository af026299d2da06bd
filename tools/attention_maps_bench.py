"""Recorded attention maps on the GPU: what the probability kernel and enable_attention_hooks cost.

One run prints the card and its power limit, then CUDA-event times (median of alternating repetitions after warm-up):
  * the stage op lseg_attn_probs at B=8, N=901 (ViT-L/16 at 480^2) and B=4, N=2117 (736^2), 16 heads: time, and the
    rate at which it writes the B*heads*N^2*4 bytes it must write, against a plain device fill of a buffer of the same
    size measured in the same run (the store bandwidth this card reaches) and the 3.35 TB/s of the H100 SXM data sheet;
  * LSegNet.predict at B=8, 480x480, K=150, on a net built with enable_attention_hooks and on one without, alternating.
Seeded synthetic weights (oracle/synth.py); one JSON line per measurement.

Usage:  python tools/attention_maps_bench.py [--reps 5] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("LSEG_ALLOW_HASH_TOKENIZER", "1")  # seeded synthetic weights: no CLIP BPE vocabulary offline

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def compare(arms, reps, iters):
    """{name: fn} -> {name: median ms per call}, the arms alternating within every repetition."""
    for fn in arms.values():  # warm-up: plans, text features, module loading
        fn()
        fn()
    torch.cuda.synchronize()
    got = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            got[k].append(time_ms(fn, iters))
    return {k: sorted(v)[len(v) // 2] for k, v in got.items()}


def report(rec):
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attention_maps_bench needs a CUDA device")
    import importlib
    importlib.import_module("lang-seg_b200")
    from lseg_b200 import ops
    from lseg_b200.lseg_net import LSegNet
    from oracle import synth

    report({"card": card()})
    heads = 16
    for B, N in ((8, 901), (4, 2117)):
        g = torch.Generator(device="cuda").manual_seed(B * N)
        qkv = torch.randn((B, N, 3 * heads * 64), generator=g, device="cuda").half()
        out = torch.empty((B, heads, N, N), device="cuda")
        fill = torch.empty_like(out)
        t = compare({"attn_probs": lambda: ops.attn_probs(qkv, heads, out=out), "fill": lambda: fill.fill_(1.0)},
                    a.reps, a.iters)
        nbytes = out.numel() * 4
        report({"case": f"attn_probs_B{B}_N{N}_h{heads}", "ms": round(t["attn_probs"], 4), "bytes": nbytes,
                "GB_s": round(nbytes / t["attn_probs"] / 1e6, 1), "fill_ms": round(t["fill"], 4),
                "fill_GB_s": round(nbytes / t["fill"] / 1e6, 1),
                "share_of_fill": round(t["fill"] / t["attn_probs"], 3),
                "share_of_3.35TB_s": round(nbytes / t["attn_probs"] / 1e-3 / HBM_PEAK, 3)})
        del qkv, out, fill

    kw = dict(backbone="clip_vitl16_384", features=256, crop_size=480, arch_option=0, block_depth=0, activation="lrelu")
    sd = synth.make_state_dict(0)
    nets = {}
    for flag in (False, True):
        n = LSegNet(labels=synth.ade20k_labels(), enable_attention_hooks=flag, **kw)
        n.load_state_dict(sd)
        nets[flag] = n.cuda().eval()
    B, H, W, K = 8, 480, 480, 150
    x = synth.make_image(B, H, W, seed=5).cuda()
    tokens = synth.tokenize(synth.ade20k_labels()[:K])
    t = compare({"predict": lambda: nets[False].predict(x, tokens),
                 "predict_hooks": lambda: nets[True].predict(x, tokens)}, a.reps, a.iters)
    n_tok = (H // 16) * (W // 16) + 1
    report({"case": f"predict_B{B}_{H}x{W}_K{K}", **{k + "_ms": round(v, 4) for k, v in t.items()},
            "extra_ms": round(t["predict_hooks"] - t["predict"], 4),
            "attention_bytes": 4 * B * heads * n_tok * n_tok * 4})


if __name__ == "__main__":
    main()
