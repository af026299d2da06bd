"""Ragged batches on the GPU: eight requests, eight label sets — what one ragged call costs next to the two ways of
serving them without it.

Workload: B=8 images at 480x480, disjoint label sets of sizes {3, 5, 12, 20, 40, 80, 150, 150} (ADE20K names, then
synthetic prompts). Arms, timed with CUDA events, alternating within every repetition after warm-up (median):
  (a) ragged:   net.predict(x, sets) and net(x, sets)
  (b) per-image: eight B=1 calls, each with its own set (predict / forward)
  (c) union:    one B=8 forward on the union of the sets, then each image's channels sliced and argmaxed in torch
The algorithmic pixel x text GEMM FLOP and fp32 logits bytes of every arm are computed from shapes. Seeded synthetic
weights (oracle/synth.py); prints the card and its power limit, then one JSON line per arm.

Usage:  python tools/ragged_bench.py [--reps 7] [--iters 5]
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

SIZES = (3, 5, 12, 20, 40, 80, 150, 150)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import lseg_b200  # noqa: F401
    from lseg_b200.lseg_net import LSegNet
    from oracle import synth

    print(json.dumps({"card": card()}), flush=True)
    net = LSegNet(labels=synth.ade20k_labels(), backbone="clip_vitl16_384", features=256, crop_size=480, arch_option=0,
                  block_depth=0, activation="lrelu")
    net.load_state_dict(synth.make_state_dict(0))
    net = net.cuda().eval()
    pool = synth.ade20k_labels() + [f"synthetic prompt {i}" for i in range(1000)]
    sets, start = [], 0
    for k in SIZES:
        sets.append(pool[start:start + k])
        start += k
    union = [name for s in sets for name in s]
    offs = [sum(SIZES[:b]) for b in range(len(SIZES))]
    B, H, W = len(SIZES), 480, 480
    x = synth.make_image(B, H, W, seed=1).cuda()

    def union_predict():
        logits = net(x, union)
        return [logits[b, o:o + k].argmax(0) for b, (o, k) in enumerate(zip(offs, SIZES))]

    def union_forward():
        logits = net(x, union)
        return [logits[b:b + 1, o:o + k] for b, (o, k) in enumerate(zip(offs, SIZES))]

    arms = {
        "ragged_predict": lambda: net.predict(x, sets),
        "ragged_forward": lambda: net(x, sets),
        "per_image_predict": lambda: [net.predict(x[b:b + 1], sets[b]) for b in range(B)],
        "per_image_forward": lambda: [net(x[b:b + 1], sets[b]) for b in range(B)],
        "union_predict": union_predict,
        "union_forward": union_forward,
    }
    # the ragged and the union results agree before anything is timed
    ragged = net(x, sets)
    for b, t in enumerate(union_forward()):
        assert t.shape == ragged[b].shape
    for fn in arms.values():  # warm-up: plans, text features, module loading
        fn()
        fn()
    torch.cuda.synchronize()
    got = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, fn in arms.items():
            got[k].append(time_ms(fn, args.iters))

    P, C = (H // 2) * (W // 2), net.out_c
    sum_k, n_union = sum(SIZES), len(union)
    gemm = {"ragged": 2.0 * P * C * sum_k, "per_image": 2.0 * P * C * sum_k, "union": 2.0 * B * P * C * n_union}
    logit_bytes = {"ragged": 4.0 * sum_k * H * W, "per_image": 4.0 * sum_k * H * W, "union": 4.0 * B * n_union * H * W}
    for k, v in got.items():
        arm = k.rsplit("_", 1)[0]
        kind = k.rsplit("_", 1)[1]
        print(json.dumps({"arm": k, "ms": round(sorted(v)[len(v) // 2], 3), "img_per_s": round(B * 1e3 / sorted(v)[len(v) // 2], 1),
                          "gemm_gflop": round(gemm[arm] / 1e9, 2),
                          "logits_gb": round(logit_bytes[arm] / 1e9, 3) if kind == "forward" or arm == "union" else 0.0,
                          "B": B, "HW": [H, W], "k": list(SIZES)}), flush=True)


if __name__ == "__main__":
    main()
