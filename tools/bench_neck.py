"""RepVGG-PluX neck at the config-2 level shapes (100x168, 50x84, 25x42, 13x21), bs=2, C=256: forward_tokens against the
reference-structured NCHW path (tokens_to_maps -> RepVGGPluXNetwork.forward in eval mode on cuDNN -> maps_to_tokens), with
torch.backends.cudnn.allow_tf32 False and True.

  python tools/bench_neck.py [--reps 20] [--rounds 3] [--out FILE]

Every call is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating
within each round.  GFLOP: torch.utils.flop_counter on the NCHW forward at these shapes (the unfolded model's work);
TFLOP/s is that over the time.  Launches: GPU kernels and memsets of one forward, counted with torch.profiler.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from collections import OrderedDict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from tools import make_neck_golden as mng  # noqa: E402

SHAPES = [(100, 168), (50, 84), (25, 42), (13, 21)]
B, C = 2, 256


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()


def timed(fn, reps, flush):
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def launches(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    net = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=4, norm_layer=torch.nn.BatchNorm2d, activation=torch.nn.SiLU)
    net.load_state_dict(mng.neck_state_dict({k: v.shape for k, v in net.state_dict().items()}, mng.NECK_SEED))
    net = net.to(dev).eval()
    g = torch.Generator().manual_seed(0)
    mem = torch.randn(B, sum(h * w for h, w in SHAPES), C, generator=g).to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def tokens():
        return net.forward_tokens(mem, SHAPES)

    def nchw():
        maps = pkg.cabi.tokens_to_maps(mem, SHAPES)
        return pkg.cabi.maps_to_tokens([f.contiguous() for f in net(OrderedDict(enumerate(maps))).values()])

    from torch.utils.flop_counter import FlopCounterMode

    with torch.no_grad():
        with FlopCounterMode(display=False) as fc:
            net(OrderedDict(enumerate(pkg.cabi.tokens_to_maps(mem, SHAPES))))
        gflop = fc.get_total_flops() / 1e9
        arms = {"forward_tokens": (tokens, None), "nchw_cudnn_fp32": (nchw, False), "nchw_cudnn_tf32": (nchw, True)}
        prev = torch.backends.cudnn.allow_tf32
        res = {k: [] for k in arms}
        n_launch, diff = {}, {}
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            for _ in range(3):
                fn()
            n_launch[name] = launches(fn)
        net64 = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=4).to(dev).double().eval()
        net64.load_state_dict(net.state_dict())
        maps64 = [m.double() for m in pkg.cabi.tokens_to_maps(mem, SHAPES)]
        want = torch.cat([f.flatten(2).transpose(1, 2) for f in net64(OrderedDict(enumerate(maps64))).values()], 1)
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            diff[name] = float((fn().double() - want).abs().max())
        for _ in range(a.rounds):
            for name, (fn, tf32) in arms.items():
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                res[name].append(timed(fn, a.reps, flush))
        torch.backends.cudnn.allow_tf32 = prev
    out = {"card": card(), "shapes": SHAPES, "batch": B, "channels": C, "gflop": round(gflop, 2), "arms": {}}
    for name in arms:
        out["arms"][name] = {"ms": [round(t, 3) for t in res[name]],
                             "tflops": [round(gflop / t, 1) for t in res[name]],
                             "launches": n_launch[name], "max_abs_err_vs_fp64": diff[name]}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
