"""Per-kernel breakdown of eager encoder-half forwards at the bench workload, from a torch.profiler trace (CUDA activities).

  python tools/profile_breakdown.py --out DIR [--steps 3]

Writes DIR/breakdown.pt.trace.json (the raw trace) and DIR/breakdown.txt: device time per step by kernel name, with the
launches made inside sdetr_ffn_fused_layernorm (the encoder FFN) also summed on their own, since the FFN may share kernel
names with other projections.  The card name and power limit are recorded at the top of the summary.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200.synthetic import build_model, make_inputs  # noqa: E402

FFN_RANGE = "sdetr_ffn_fused_layernorm"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the summary still states that the card is unknown
        return f"unknown ({type(e).__name__})"


def summarize(trace_path, steps):
    ev = json.load(open(trace_path))["traceEvents"]
    ffn_ranges = collections.defaultdict(list)  # tid -> [(ts, end)] of the FFN entry point on the host
    launch_at = {}                              # correlation id -> (tid, ts) of the runtime launch call
    for e in ev:
        if e.get("ph") != "X":
            continue
        if e.get("cat") == "user_annotation" and e.get("name") == FFN_RANGE:
            ffn_ranges[e["tid"]].append((e["ts"], e["ts"] + e["dur"]))
        elif e.get("cat") in ("cuda_runtime", "cuda_driver") and "correlation" in e.get("args", {}):
            launch_at[e["args"]["correlation"]] = (e["tid"], e["ts"])
    tot, cnt, ffn_tot, ffn_cnt = collections.Counter(), collections.Counter(), collections.Counter(), collections.Counter()
    for e in ev:
        if e.get("ph") != "X" or e.get("cat") != "kernel":
            continue
        name = re.sub(r"^void ", "", re.sub(r"\(.*", "", e["name"]))[:90]
        tot[name] += e["dur"]
        cnt[name] += 1
        tid, ts = launch_at.get(e.get("args", {}).get("correlation"), (None, None))
        if tid is not None and any(a <= ts <= b for a, b in ffn_ranges.get(tid, ())):
            ffn_tot[name] += e["dur"]
            ffn_cnt[name] += 1
    s, f = sum(tot.values()), sum(ffn_tot.values())
    lines = [f"card: {card()}",
             f"device time per step {s / steps:.1f} us over {sum(cnt.values()) / steps:.0f} launches "
             f"(eager, {steps} steps, kernels serialised on one stream; profiler on)",
             f"encoder FFN (launches inside {FFN_RANGE}): {f / steps:.1f} us per step, {100 * f / max(s, 1e-9):.1f}% of device time, "
             f"{sum(ffn_cnt.values()) / steps:.0f} launches"]
    for k, v in sorted(ffn_tot.items(), key=lambda x: -x[1]):
        lines.append(f"  FFN {v / steps:9.1f} us {100 * v / s:5.1f}% x{ffn_cnt[k] / steps:4.0f}  {k}")
    lines.append("all kernels:")
    for k, v in sorted(tot.items(), key=lambda x: -x[1])[:40]:
        lines.append(f"{v / steps:9.1f} us {100 * v / s:5.1f}% x{cnt[k] / steps:4.0f}  {k}")
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--workload", default="resnet50_800_1333_bs2")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    model = build_model().to(dev)
    feats, masks, pos = make_inputs(args.workload, seed=0, device=dev)
    orig = pkg.cabi.ffn_fused_layernorm

    def ffn(*a, **k):
        with torch.profiler.record_function(FFN_RANGE):
            return orig(*a, **k)

    pkg.cabi.ffn_fused_layernorm = ffn
    try:
        with torch.no_grad():
            plan = model.make_plan(masks)
            for _ in range(3):
                model.forward_encoder(feats, masks, pos, plan=plan)
            torch.cuda.synchronize()
            acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
            with torch.profiler.profile(activities=acts) as prof:
                for _ in range(args.steps):
                    model.forward_encoder(feats, masks, pos, plan=plan)
                torch.cuda.synchronize()
    finally:
        pkg.cabi.ffn_fused_layernorm = orig
    trace = os.path.join(args.out, "breakdown.pt.trace.json")
    prof.export_chrome_trace(trace)
    text = summarize(trace, args.steps)
    open(os.path.join(args.out, "breakdown.txt"), "w").write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
