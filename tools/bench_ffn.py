"""Encoder FFN + LayerNorm: the fused entry point (sdetr_ffn_fused_layernorm) against the two-GEMM composition it replaced
(gemm_f16x3_pre for linear1, again with the ReLU fused for linear2, then add_layernorm), at the six encoder layers' row
counts of the bench workload (salience_detr_resnet50_800_1333, bs=2), hidden 2048.

  python tools/bench_ffn.py [--reps 20] [--out FILE]

Each call is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians.  TFLOP/s counts what the tensor
cores execute: 3 fp16 products per logical product (3xFP16).  The fused kernel keeps x and the hidden activations on chip and
streams all of W1 and W2 (fp16 hi / lo pairs, 4 MiB at hidden 2048) from L2 once per 128-row panel; weight_bytes is that
traffic and fused_l2_gbps its rate, to set against the L2 ceiling of tools/micro/l2_bw.cu.  Also reports whether, on one CTA per panel (cap 1), the
fused linear2 output before LayerNorm equals the two-GEMM path's bit for bit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402

ROWS = (22726, 18180, 13634, 13634, 9090, 4544)
HIDDEN = 2048
PANEL_ROWS = 128  # rows per panel of the fused kernel (kFM in csrc/ffn_fused.cu)


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()


def timed(fn, reps, flush):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1000.0)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    cabi = pkg.cabi
    g = torch.Generator().manual_seed(0)
    w1 = (torch.randn(HIDDEN, 256, generator=g) / 16).to(dev)
    b1 = torch.randn(HIDDEN, generator=g).to(dev)
    w2 = (torch.randn(256, HIDDEN, generator=g) / HIDDEN ** 0.5).to(dev)
    b2 = torch.randn(256, generator=g).to(dev)
    gamma = (1 + 0.1 * torch.randn(256, generator=g)).to(dev)
    beta = (0.1 * torch.randn(256, generator=g)).to(dev)
    s1, s2 = cabi.split_f16_pair(w1), cabi.split_f16_pair(w2)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    res = {"card": card(), "hidden": HIDDEN, "reps": args.reps, "shapes": []}
    tot_f = tot_t = tot_w = 0.0
    for rows in ROWS:
        x = torch.randn(rows, 256, generator=g).to(dev)
        y = torch.empty_like(x)
        h = torch.empty(rows, HIDDEN, device=dev)
        pbuf = torch.empty_like(x)

        def fused():
            cabi.ffn_fused_layernorm(x, s1, b1, s2, b2, gamma, beta, 1e-5, out=y)

        def two():
            cabi.gemm_f16x3_pre(x, *s1, b1, 0, out=h)
            cabi.gemm_f16x3_pre(h, *s2, b2, 1, out=pbuf)
            cabi.add_layernorm(x, pbuf, gamma, beta, 1e-5, out=y)

        t_f, t_t = timed(fused, args.reps, flush), timed(two, args.reps, flush)
        exe = 3 * 2 * 2 * rows * 256 * HIDDEN  # executed tensor-core flops: 3 products x 2 GEMMs
        wbytes = -(-rows // PANEL_ROWS) * 2 * 2 * HIDDEN * 256 * 2  # per panel: W1 and W2, hi and lo, fp16
        tot_f, tot_t, tot_w = tot_f + t_f, tot_t + t_t, tot_w + wbytes
        res["shapes"].append({"rows": rows, "fused_us": round(t_f, 1), "two_gemm_us": round(t_t, 1),
                              "fused_tflops_executed": round(exe / t_f / 1e6, 1),
                              "two_gemm_tflops_executed": round(exe / t_t / 1e6, 1),
                              "weight_bytes": wbytes, "fused_l2_gbps": round(wbytes / t_f / 1e3)})
        print(json.dumps(res["shapes"][-1]), flush=True)
    res["fused_us_total"], res["two_gemm_us_total"] = round(tot_f, 1), round(tot_t, 1)
    res["fused_vs_two_gemm"] = round(tot_f / tot_t, 4)
    res["weight_bytes_total"], res["fused_l2_gbps"] = int(tot_w), round(tot_w / tot_f / 1e3)
    lib = cabi.lib()
    x = torch.randn(1000, 256, generator=g).to(dev)
    lib.sdetr_set_persistent_ctas(1)
    try:
        res["cap1_bare_equals_two_gemm_bitwise"] = bool(torch.equal(
            cabi.ffn_fused_layernorm(x, s1, b1, s2, b2), cabi.gemm_f16x3_pre(cabi.gemm_f16x3_pre(x, *s1, b1, 0), *s2, b2, 1)))
    finally:
        lib.sdetr_set_persistent_ctas(0)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
