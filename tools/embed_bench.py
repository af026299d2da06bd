"""Encode once / query many on the GPU: what a query on a stored pixel embedding costs next to the calls it replaces.

One run prints the card and its power limit, then CUDA-event times (median of alternating repetitions after warm-up):
  * B=8, 480x480, K in {2, 150, 512}: forward vs encode_image + query, and predict vs a query with a mask output;
  * PixelEmbedding.features(): time and achieved bandwidth against the H100 SXM's 3.35 TB/s;
  * the multi-scale evaluator on a 512x683 image: evaluator(image, L) vs encode once + evaluator(embedding, L).
Seeded synthetic weights (oracle/synth.py); one JSON line per measurement.

Usage:  python tools/embed_bench.py [--reps 5] [--iters 10]
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
        raise SystemExit("embed_bench needs a CUDA device")
    import importlib
    importlib.import_module("lang-seg_b200")
    from lseg_b200.evaluator import MultiScaleEvaluator
    from lseg_b200.lseg_net import LSegNet
    from oracle import synth

    report({"card": card()})
    net = LSegNet(labels=synth.ade20k_labels(), backbone="clip_vitl16_384", features=256, crop_size=480, arch_option=0,
                  block_depth=0, activation="lrelu")
    net.load_state_dict(synth.make_state_dict(0))
    net = net.cuda().eval()
    B, H, W = 8, 480, 480
    x = synth.make_image(B, H, W, seed=5).cuda()
    emb = net.encode_image(x)
    for K in (2, 150, 512):
        tokens = synth.tokenize(synth.ade20k_labels()[:K]) if K <= 150 else synth.synthetic_prompts(K, seed=0)
        out = torch.empty((B, K, H, W), device="cuda")
        t = compare({"forward": lambda: net(x, tokens, out=out),
                     "encode_image": lambda: net.encode_image(x),
                     "query": lambda: net(emb, tokens, out=out),
                     "predict": lambda: net.predict(x, tokens),
                     "query_mask": lambda: net.predict(emb, tokens)}, a.reps, a.iters)
        report({"case": f"B{B}_{H}x{W}_K{K}", **{k + "_ms": round(v, 4) for k, v in t.items()},
                "forward_over_query": round(t["forward"] / t["query"], 2),
                "predict_over_query_mask": round(t["predict"] / t["query_mask"], 2)})

    t = compare({"features": lambda: emb.features()}, a.reps, a.iters)["features"]
    C, P = emb.out_c, (H // 2) * (W // 2)
    nbytes = B * P * (2 * C + 4 * (C // 32) + 4 * C)
    report({"case": f"features_B{B}_{H}x{W}", "ms": round(t, 4), "bytes": nbytes, "GB_s": round(nbytes / t / 1e6, 1),
            "share_of_3.35TB_s": round(nbytes / t / 1e-3 / HBM_PEAK, 3)})
    del emb

    ev = MultiScaleEvaluator(net)
    img = synth.make_image(1, 512, 683, seed=683).cuda()
    labels = synth.ade20k_labels()
    enc = ev.encode(img)
    torch.cuda.synchronize()
    t = compare({"evaluator_image": lambda: ev(img, labels), "evaluator_embedding": lambda: ev(enc, labels)},
                max(1, a.reps // 2), 2)
    t_enc = compare({"encode": lambda: ev.encode(img)}, 1, 2)["encode"]
    report({"case": "evaluator_512x683_K150", "crops": ev.num_forwards(img)[1], **{k + "_ms": round(v, 3) for k, v in t.items()},
            "encode_ms": round(t_enc, 3), "image_over_embedding": round(t["evaluator_image"] / t["evaluator_embedding"], 2)})


if __name__ == "__main__":
    main()
