#!/usr/bin/env python
"""Time each distinct GEMM shape / epilogue of the B=8, 480x480 LSeg ViT-L forward through ops.gemm.

Each shape runs on seeded random operands (the timing does not depend on the values), warmed up, then timed with CUDA
events over enough back-to-back launches to fill at least --min-ms; the median of --reps such windows is reported as
ms per launch and TFLOP/s (2 M N K taps over that time). Every shape is timed twice in the same process, with 2-CTA
clusters wherever possible and with every GEMM unclustered (lseg_debug_set_gemm_cluster modes 3 and 1), the two windows
alternating; "cl" is the cluster size the planner picks for the shape by default. The card name and its power limit are
printed first: the numbers are only meaningful with them.

LSEG_GEMM_PROBE (read once per process, see GemmParams::probe) turns parts of the kernel off; run the script once
without it and once with LSEG_GEMM_PROBE=1 (epilogue skipped) to see how much of each shape's time the epilogue adds.

    python tools/gemm_shapes.py [--min-ms 50] [--reps 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lseg_b200  # noqa: E402,F401
from lseg_b200 import ops  # noqa: E402

B, IMG = 8, 480
TOKENS = B * ((IMG // 16) ** 2 + 1)     # ViT-L/16 rows: 8 x 901
LEVELS = [(120, 256), (60, 512), (30, 1024), (15, 1024)]  # decoder level side, reassembled channels (layerN_rn input)
FEAT, OUT_C, LABELS = 256, 512, 150
PIX = B * (IMG // 2) ** 2               # head1 / pixel x text rows


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def shapes(g):
    """(name, flops, gemm args, gemm keywords) per shape; every launch writes only buffers allocated here."""
    dev = "cuda"
    h = lambda *s: (torch.randn(*s, generator=g, device=dev) * 0.5).half()  # noqa: E731
    f = lambda *s: torch.randn(*s, generator=g, device=dev)  # noqa: E731
    out = []

    def linear(name, M, K, N, **kw):
        a, w, bias = h(M, K), ops.pad_rows(h(N, K) * 0.05), f(N)
        out.append((name, 2.0 * M * N * K, (a, w, N), dict(M=M, bias=bias, **kw)))

    x = f(TOKENS, 1024)
    linear("vit qkv      1024->3072 f16", TOKENS, 1024, 3072, out_f16=torch.empty(TOKENS, 3072, device=dev).half())
    linear("vit proj     1024->1024 +=x", TOKENS, 1024, 1024, res_f32=x, out_f32=x)
    linear("vit fc1      1024->4096 gelu", TOKENS, 1024, 4096, act=ops.ACT_GELU,
           out_f16=torch.empty(TOKENS, 4096, device=dev).half())
    linear("vit fc2      4096->1024 +=x", TOKENS, 4096, 1024, res_f32=x, out_f32=x)

    for side, cin in LEVELS:
        px = B * side * side
        xin = h(B, side, side, cin)
        wrn = ops.pad_rows(h(FEAT, 9 * cin) * 0.02)
        o32, r16 = torch.empty(px, FEAT, device=dev), torch.empty(px, FEAT, device=dev).half()
        out.append((f"layer_rn {side:3d}^ {cin:4d}->256 f32+relu", 2.0 * px * FEAT * 9 * cin, (xin, wrn, FEAT),
                    dict(conv=(3, 1), out_f32=o32, out_f16_relu=r16, ldc=FEAT)))
        t = h(B, side, side, FEAT)
        w3 = ops.pad_rows(h(FEAT, 9 * FEAT) * 0.02)
        sc, sh = f(FEAT).abs() + 0.5, f(FEAT)
        res, t16 = f(px, FEAT), torch.empty(px, FEAT, device=dev).half()
        s32, s16 = torch.empty(px, FEAT, device=dev), torch.empty(px, FEAT, device=dev).half()
        fl = 2.0 * px * FEAT * 9 * FEAT
        out.append((f"rcu conv1 {side:3d}^ bn relu f16", fl, (t, w3, FEAT),
                    dict(conv=(3, 1), scale=sc, bias=sh, act=ops.ACT_RELU, out_f16=t16, ldc=FEAT)))
        out.append((f"rcu conv2 {side:3d}^ bn +res f32+relu", fl, (t, w3, FEAT),
                    dict(conv=(3, 1), scale=sc, bias=sh, res_f32=res, out_f32=s32, out_f16_relu=s16, ldc=FEAT)))
        a1, w1, b1 = h(px, FEAT), ops.pad_rows(h(FEAT, FEAT) * 0.05), f(FEAT)
        out.append((f"out_conv  {side:3d}^ 1x1 f32", 2.0 * px * FEAT * FEAT, (a1, w1, FEAT), dict(bias=b1, out_f32=o32)))

    path, wh, bh = h(PIX, FEAT), ops.pad_rows(h(OUT_C, FEAT) * 0.05), f(OUT_C)
    feat16 = torch.empty(PIX, OUT_C, device=dev).half()
    sumsq = torch.empty(PIX, OUT_C // 32, device=dev)
    out.append(("head1     256->512 f16+sumsq", 2.0 * PIX * OUT_C * FEAT, (path, wh, OUT_C),
                dict(bias=bh, out_f16=feat16, out_row_sumsq=sumsq)))
    text = ops.pad_rows(h(LABELS, OUT_C) * 0.05)
    logits = torch.empty(B, LABELS, PIX // B, device=dev).half()
    ss = f(PIX, OUT_C // 32).abs() + 1.0
    out.append(("pixel x text 512->150 nchw", 2.0 * PIX * LABELS * OUT_C, (feat16, text, LABELS),
                dict(out_f16=logits, store=ops.STORE_NCHW_T, nchw=(PIX // B, LABELS), row_sumsq=ss, row_scale=14.0)))
    return out


def window(fn, n):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / n


def time_launch(fn, min_ms, reps):
    """Median ms per launch with pairs wherever possible (mode 3) and unclustered (mode 1), the windows alternating."""
    times = {3: [], 1: []}
    for mode in times:
        ops.set_gemm_cluster(mode)
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    n = max(5, int(min_ms / max(window(fn, 5), 1e-3)) + 1)
    for _ in range(reps):
        for mode, t in times.items():
            ops.set_gemm_cluster(mode)
            t.append(window(fn, n))
    ops.set_gemm_cluster(2)
    return {mode: sorted(t)[len(t) // 2] for mode, t in times.items()}, n


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--min-ms", type=float, default=50.0, help="least timed window per repetition (ms)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_shapes.py needs a CUDA device")
    name, power = card()
    probe = os.environ.get("LSEG_GEMM_PROBE", "0")
    print(f"# {name}, power limit / max SM clock: {power}; LSEG_GEMM_PROBE={probe}")
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    print(f"{'shape':40s} cl {'paired ms':>9s} {'TFLOP/s':>8s} | unclustered {'ms':>9s} {'TFLOP/s':>8s}")
    for label, flops, gargs, kw in shapes(g):
        cl = ops.gemm_cluster(*gargs, **kw)["cluster"]
        ms, n = time_launch(lambda: ops.gemm(*gargs, **kw), args.min_ms, args.reps)
        tf = {mode: flops / (t * 1e-3) / 1e12 for mode, t in ms.items()}
        rows.append({"shape": label, "cluster": cl, "ms_paired": ms[3], "tflops_paired": tf[3], "ms_unclustered": ms[1],
                     "tflops_unclustered": tf[1], "launches": n})
        print(f"{label:40s} {cl:2d} {ms[3]:9.4f} {tf[3]:8.1f} | {'':11s} {ms[1]:9.4f} {tf[1]:8.1f}  "
              f"({n} launches per window, {ms[1] / ms[3] - 1:+.1%})")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": name, "power": power, "probe": probe, "shapes": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
