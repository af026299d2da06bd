"""Cost of scoring LSeg's output with the on-device metric counters (lseg_b200.metrics) against the host-side scoring of
PyTorch-Encoding's SegmentationMetric (torch.max -> int64 mask to the host -> numpy histograms).

Prints the card name and its power limit first, then, each over `--reps` timed repetitions (median and min..max):
  1. batch 8 x 480x480, K = 150 (random-init ViT-L/16 weights): predict() + the encoding-style numpy metric of the mask,
     against update_metric() (fused argmax + counters, nothing leaves the GPU);
  2. predict() alone against update_metric(): the cost of the histogram epilogue over the mask store, at K = 150 and at
     K = nclass = 2 (the zero-shot shape, where the block histogram's atomics share the fewest addresses);
  3. SegmentationMetric.update on one [1,150,512,683] fp32 evaluator output, with the bytes it must read (scores + int64
     target) over its time.
Every timed region ends in a device synchronise (the numpy side needs the mask on the host anyway).

    python tools/seg_metrics_bench.py [--reps 20]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def fmt(t):
    return f"{t[0]:8.3f} ms  ({t[1]:.3f} .. {t[2]:.3f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_metrics_bench needs a CUDA device")
    name, power = card()
    print(f"card: {name}, power limit / max SM clock: {power}")

    import lseg_b200  # noqa: F401
    from lseg_b200 import tokenizer
    from lseg_b200.lseg_net import LSegNet
    from lseg_b200.metrics import SegmentationMetric
    from segstats_oracle import EncodingMetric
    tokenizer.enable_stand_in()  # random-init weights: no CLIP vocabulary offline
    labels = [f"label {i}" for i in range(150)]
    net = LSegNet(labels=labels, backbone="clip_vitl16_384", features=256, crop_size=480, arch_option=0, block_depth=0,
                  activation="lrelu").cuda().eval()
    B, S, K = 8, 480, 150
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, 3, S, S, device="cuda", generator=g)
    target = torch.randint(-1, K, (B, S, S), device="cuda", generator=g)
    target_host = target.cpu().numpy()
    enc = EncodingMetric(K)
    metric = SegmentationMetric(K)

    def host_path():
        mask = net.predict(x).cpu().numpy()
        enc.update(target_host, mask)

    def fused_path():
        net.update_metric(metric, x, target)

    def predict_only():
        net.predict(x)

    # alternate the variants so that drift of the shared host affects all of them alike
    res = {"host": [], "fused": [], "predict": []}
    for _ in range(3):
        res["host"].append(timed(host_path, max(1, args.reps // 3)))
        res["fused"].append(timed(fused_path, max(1, args.reps // 3)))
        res["predict"].append(timed(predict_only, max(1, args.reps // 3)))
    for k in res:
        med = sorted(r[0] for r in res[k])[1]
        res[k] = (med, min(r[1] for r in res[k]), max(r[2] for r in res[k]))
    print(f"config 2 (B={B}, {S}x{S}, K={K}), per step (median of 3 rounds, min .. max over all reps):")
    print(f"  predict() + numpy encoding metric : {fmt(res['host'])}")
    print(f"  update_metric() (fused)           : {fmt(res['fused'])}")
    print(f"  predict() alone (mask store only) : {fmt(res['predict'])}")
    print(f"  histogram epilogue over mask store: {res['fused'][0] - res['predict'][0]:+.3f} ms (medians)")

    # K = nclass = 2 (the zero-shot shape): every counted pixel lands on one of 6 shared-memory bins per block, the
    # worst case for same-address atomics in the fused epilogue
    pair = ["others", "cat"]
    m_pair = SegmentationMetric(2)
    t_pair = torch.randint(-1, 2, (B, S, S), device="cuda", generator=g)
    res2 = {"fused": [], "predict": []}
    for _ in range(3):
        res2["fused"].append(timed(lambda: net.update_metric(m_pair, x, t_pair, pair), max(1, args.reps // 3)))
        res2["predict"].append(timed(lambda: net.predict(x, pair), max(1, args.reps // 3)))
    for k in res2:
        med = sorted(r[0] for r in res2[k])[1]
        res2[k] = (med, min(r[1] for r in res2[k]), max(r[2] for r in res2[k]))
    print(f"K = nclass = 2 (B={B}, {S}x{S}), per step:")
    print(f"  update_metric() (fused)           : {fmt(res2['fused'])}")
    print(f"  predict() alone (mask store only) : {fmt(res2['predict'])}")
    print(f"  histogram epilogue over mask store: {res2['fused'][0] - res2['predict'][0]:+.3f} ms (medians)")

    out = torch.randn(1, 150, 512, 683, device="cuda", generator=g)
    t1 = torch.randint(-1, 150, (512, 683), device="cuda", generator=g)
    m2 = SegmentationMetric(150)
    t = timed(lambda: m2.update(t1, out), args.reps * 5)
    nbytes = out.numel() * 4 + t1.numel() * 8
    print(f"SegmentationMetric.update [1,150,512,683] fp32: {fmt(t)}, {nbytes / 1e6:.1f} MB read "
          f"-> {nbytes / (t[0] * 1e-3) / 1e9:.0f} GB/s (median)")
    # same scores, numpy side: torch.max on the GPU, mask to the host, encoding's histograms
    t1h = t1.cpu().numpy()
    e2 = EncodingMetric(150)
    th = timed(lambda: e2.update(t1h, torch.max(out, 1)[1].cpu().numpy()), args.reps)
    print(f"torch.max + numpy encoding metric, same output  : {fmt(th)}")


if __name__ == "__main__":
    main()
