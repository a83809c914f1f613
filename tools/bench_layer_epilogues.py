"""Per-layer timing of the encoder layer's two fused GEMM epilogues against the unfused pairs they replace, at the six
encoder layers' row counts of the bench workload (bs = 2):

* score:   sdetr_gemm_f16x3_pre (R x 91 logits) + sdetr_class_max_times_fg   vs   sdetr_gemm_f16x3_rowmax
* norm1:   sdetr_gemm_f16x3_pre (R x 256 output projection) + sdetr_add_layernorm(q, ., out=q)
           vs   sdetr_gemm_f16x3_add_layernorm

  python tools/bench_layer_epilogues.py [--rounds 30]

Old and new run in alternating rounds, L2 flushed before each timed call, so both read their operands from HBM as in the
step.  Per shape: median µs of each, and the HBM bytes each has to move (operands read once, results written once:
A, W pair, residual / row scale in; logits or projection out and back in for the pair).  The card's name and power limit
are printed with the numbers.
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402

LAYER_ROWS = (22726, 18180, 13634, 13634, 9090, 4544)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the output still states that the card is unknown
        return f"unknown ({type(e).__name__})"


def timed(fn, flush):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_layer_epilogues.py needs a GPU")
    dev = torch.device("cuda:0")
    cabi = pkg.cabi
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"card: {card()}")
    print(f"{'call':8s} {'R':>6s} {'old us':>8s} {'new us':>8s} {'old MB':>7s} {'new MB':>7s} {'saved us':>8s}")
    tot_old = tot_new = 0.0
    for j, R in enumerate(LAYER_ROWS):
        g = torch.Generator().manual_seed(j)
        x = torch.randn(R, 256, generator=g).to(dev)
        ws, bs = (torch.randn(91, 256, generator=g) / 16).to(dev), torch.randn(91, generator=g).to(dev)
        wo, bo = (torch.randn(256, 256, generator=g) / 16).to(dev), torch.randn(256, generator=g).to(dev)
        fg = torch.rand(R, generator=g).to(dev)
        q0 = torch.randn(R, 256, generator=g).to(dev)
        gam, bet = torch.ones(256, device=dev), torch.zeros(256, device=dev)
        sp, op = cabi.split_f16_pair(ws), cabi.split_f16_pair(wo)
        q = q0.clone()
        cases = {
            "score": (lambda: cabi.class_max_times_fg(cabi.gemm_f16x3_pre(x, *sp, bs), fg),
                      lambda: cabi.gemm_f16x3_rowmax(x, *sp, bs, fg),
                      # A + W pair + fg in, mc out; the pair also writes and reads the R x 92 padded logits
                      R * 256 * 4 + 91 * 256 * 4 + 2 * R * 4, 2 * R * 92 * 4),
            "norm1": (lambda: cabi.add_layernorm(q, cabi.gemm_f16x3_pre(x, *op, bo), gam, bet, out=q),
                      lambda: cabi.gemm_f16x3_add_layernorm_(q, x, *op, bo, gam, bet),
                      # A + W pair + q in, q out; the pair also writes and reads the R x 256 projection
                      R * 256 * 4 + 256 * 256 * 4 + 2 * R * 256 * 4, 2 * R * 256 * 4),
        }
        for name, (old, new, base_bytes, extra) in cases.items():
            for _ in range(3):
                old(), new()
            to, tn = [], []
            for _ in range(args.rounds):
                to.append(timed(old, flush))
                tn.append(timed(new, flush))
            mo, mn = statistics.median(to), statistics.median(tn)
            tot_old, tot_new = tot_old + mo, tot_new + mn
            print(f"{name:8s} {R:6d} {mo:8.1f} {mn:8.1f} {(base_bytes + extra) / 1e6:7.1f} {base_bytes / 1e6:7.1f} "
                  f"{mo - mn:8.1f}")
    print(f"sum over the six layers: old {tot_old:.1f} us, new {tot_new:.1f} us, saved {tot_old - tot_new:.1f} us")


if __name__ == "__main__":
    main()
