"""Cost of the validation loss + metric step with the fused device loss (LSegNet.loss with metric=) against the
materialising path of the reference's validation_step (net(x) -> F.cross_entropy -> metric.update on the fp32 logits).

Prints the card name and its power limit first, then per shape (B=8 480x480 K=150, and config 5's B=4 736x736 K=512),
alternating the two arms over `--rounds` rounds of `--reps` timed steps each:
  (a) logits = net(x); F.cross_entropy(logits, target, ignore_index=-1); metric.update(target, logits)
  (b) net.loss(x, target, metric=m)
the median ms per step (min .. max), each arm's torch.cuda.max_memory_allocated over its steps, the two losses and
their difference against the derived bound (tests/xent_oracle.py) of the device loss. Every timed step ends in a device
synchronise.

    python tools/xent_bench.py [--reps 10] [--rounds 3]
"""
import argparse
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

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


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("xent_bench needs a CUDA device")
    name, power = card()
    print(f"card: {name}, power limit / max SM clock: {power}")

    import lseg_b200  # noqa: F401
    from lseg_b200 import tokenizer
    from lseg_b200.lseg_net import LSegNet
    from lseg_b200.metrics import SegmentationMetric
    from xent_oracle import mean_bound
    tokenizer.enable_stand_in()  # random-init weights: no CLIP vocabulary offline

    for B, S, K in ((8, 480, 150), (4, 736, 512)):
        labels = [f"label {i}" for i in range(K)]
        net = LSegNet(labels=labels, backbone="clip_vitl16_384", features=256, crop_size=S, arch_option=0,
                      block_depth=0, activation="lrelu").cuda().eval()
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(B, 3, S, S, device="cuda", generator=g)
        target = torch.randint(-1, K, (B, S, S), device="cuda", generator=g)
        m_a, m_b = SegmentationMetric(K), SegmentationMetric(K)
        out = {}

        def arm_a():
            logits = net(x)
            out["a"] = F.cross_entropy(logits, target, ignore_index=-1)
            m_a.update(target, logits)

        def arm_b():
            out["b"] = net.loss(x, target, metric=m_b)

        arms = {"a": arm_a, "b": arm_b}
        times = {"a": [], "b": []}
        peak = {"a": 0, "b": 0}
        for fn in arms.values():  # warm-up: plans, text features, allocator
            fn()
            fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for k, fn in arms.items():
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                times[k] += timed(fn, args.reps)
                peak[k] = max(peak[k], torch.cuda.max_memory_allocated())
        logits = net(x)
        bound = mean_bound(logits.cpu().numpy(), target.cpu().numpy(), -1)
        la, lb = out["a"].item(), out["b"].item()
        print(f"B={B}, {S}x{S}, K={K} ({args.rounds} rounds x {args.reps} steps, arms alternating):")
        for k, what in (("a", "net(x) + F.cross_entropy + metric.update"), ("b", "net.loss(x, target, metric=m)")):
            ts = sorted(times[k])
            print(f"  ({k}) {what:42s}: {ts[len(ts) // 2]:8.3f} ms/step ({ts[0]:.3f} .. {ts[-1]:.3f}), "
                  f"max_memory_allocated {peak[k] / 2 ** 30:.2f} GiB")
        print(f"  loss (a) {la:.7f}  (b) {lb:.7f}  |a - b| {abs(la - lb):.3e}  bound of (b) {bound:.3e}  "
              f"agree within 2 x bound: {abs(la - lb) <= 2 * bound}")
        ca, cb = m_a.stats, m_b.stats
        print(f"  metric counters equal: {bool(torch.equal(ca, cb))}")
        del net, logits
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
