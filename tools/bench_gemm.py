"""Per-shape timing of the dense projections of one bench step, through the route the step takes (``gemm.linear`` in
MODE "auto": the 3xFP16 wgmma kernel ``gemm3x_kernel<true, false>`` for every shape here).

  python tools/bench_gemm.py [--reps 20] [--save DIR]

The shapes are the calls of one encoder-half forward at the bench workload (bs = 2, Nv = 22323 tokens per image, layer
rows 22726 / 18180 / 13634 / 13634 / 9090 / 4544) that have more than ``gemm.SMALL_M`` rows: the value projection of all
six layers in one call, enc_output, the MaskPredictor GEMMs of the two large levels, and per layer the class-score,
sampling-offset/attention and output projections.  L2 is flushed before each timed call, so every call reads its operands
from HBM as it does in the step.  Per shape: median µs, executed TFLOP/s (three MMA passes over the padded 128 x 128
tiles, the work the tensor cores do) and output GB/s; then the sums for the per-layer group and for the whole step.

``--save DIR`` writes each shape's output, from inputs seeded per shape, as DIR/<name>.npy, so that the outputs of two
builds of the library can be compared bit for bit.
"""
import argparse
import math
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402

LAYER_ROWS = (22726, 18180, 13634, 13634, 9090, 4544)
SHAPES = ([("value_proj x6", 44646, 256, 1536, None), ("enc_output", 44646, 256, 256, None)] +
          [(f"mask_pred l{lv} {part}", M, K, N, act) for lv, M in enumerate((33600, 8400))
           for part, K, N, act in (("fc", 256, 256, None), ("l2a", 256, 128, None), ("l2b", 128, 64, "gelu"),
                                   ("l2c", 64, 1, "gelu"))] +
          [(f"L{j} {part}", M, 256, N, None) for j, M in enumerate(LAYER_ROWS)
           for part, N in (("mcsp", 91), ("proj", 384), ("out_proj", 256))])


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the output still states that the card is unknown
        return f"unknown ({type(e).__name__})"


def executed_flop(M, K, N):
    return 2 * 3 * math.ceil(M / 128) * 128 * math.ceil(N / 128) * 128 * K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--save", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py needs a GPU")
    dev = torch.device("cuda:0")
    pkg.gemm.MODE = "auto"
    if args.save:
        os.makedirs(args.save, exist_ok=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"card: {card()}")
    print(f"{'gemm':20s} {'M':>6s} {'K':>4s} {'N':>5s} {'us':>8s} {'exec TF/s':>9s} {'out GB/s':>8s}")
    tot = layer = 0.0
    for i, (name, M, K, N, act) in enumerate(SHAPES):
        g = torch.Generator().manual_seed(1000 + i)
        x = torch.randn(M, K, generator=g).to(dev)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        b = torch.randn(N, generator=g).to(dev)
        run = lambda: pkg.gemm.linear(x, w, b, input_act=act)  # noqa: E731
        for _ in range(3):
            y = run()
        ts = []
        for _ in range(args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1000)
        us = statistics.median(ts)
        tot += us
        layer += us if name.startswith("L") else 0.0
        print(f"{name:20s} {M:6d} {K:4d} {N:5d} {us:8.1f} {executed_flop(M, K, N) / us / 1e6:9.1f} "
              f"{M * N * 4 / us / 1e3:8.1f}")
        if args.save:
            np.save(os.path.join(args.save, name.replace(" ", "_") + ".npy"), y.cpu().numpy())
    print(f"sum per-layer group (18 calls): {layer:.1f} us")
    print(f"sum step ({len(SHAPES)} calls): {tot:.1f} us")


if __name__ == "__main__":
    main()
