"""RepVGG-PluX neck training step at the config-2 level shapes (100x168, 50x84, 25x42, 13x21), bs=2, C=256, train mode: one
forward + backward of sum(out * R) for a fixed random R, with forward_tokens against the reference-structured NCHW path
(split -> NCHW -> RepVGGPluXNetwork.forward on cuDNN -> concatenate, the differentiable round trip
SalienceTransformer.forward takes in training) with torch.backends.cudnn.allow_tf32 False and True.

  python tools/bench_neck_train.py [--reps 10] [--rounds 3] [--out FILE]

Every step is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating
within each round.  Each arm runs eagerly and as the replay of a CUDA graph of the same step (the *_graph arms): the eager
token step issues ~1800 launches and is bound by the host, the replay by the device.  Also per arm: launches per step (GPU kernels and memsets, torch.profiler), host synchronisations per step
(torch.cuda.set_sync_debug_mode("warn")), peak memory of a step, and the max |error| of the output, grad(memory) and the
convolution weight gradients against a float64 run of forward().  A separate profiled run of the token arm gives the share of
GPU time per kernel family.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings
from collections import OrderedDict, defaultdict

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


def family(name):
    """kernel family of a GPU kernel name, for the profile breakdown"""
    n = name.lower()
    for key, fam in (("conv_wgrad_f16x3", "new: conv weight gradient"), ("wgrad_reduce", "new: conv weight gradient"),
                     ("conv_f16x3_kernel<true>", "new: stride-2 input gradient (transposed conv)"),
                     ("upsample_concat_backward", "new: upsample backward"),
                     ("conv_f16x3_kernel", "conv_f16x3: forward and stride-1 input gradient"),
                     ("pow2", "scales and fp16 splits"), ("split_f16", "scales and fp16 splits"),
                     ("upsample_concat", "upsample-concat forward"),
                     ("batch_norm", "torch BatchNorm"), ("bn_", "torch BatchNorm"), ("silu", "torch SiLU"),
                     ("softmax", "torch context gate"), ("gemm", "torch context gate"), ("sigmoid", "torch context gate"),
                     ("cat", "torch concatenations"), ("memset", "memsets")):
        if key in n:
            return fam
    return "other torch ops"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    net = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=4, norm_layer=torch.nn.BatchNorm2d, activation=torch.nn.SiLU)
    net.load_state_dict(mng.neck_state_dict({k: v.shape for k, v in net.state_dict().items()}, mng.NECK_SEED))
    net = net.to(dev).train()
    params = list(net.parameters())
    conv_w = [p for n, p in net.named_parameters() if p.dim() == 4 and p.shape[-1] in (1, 3) and "se_module" not in n
              and "conv_mask" not in n]
    g = torch.Generator().manual_seed(0)
    mem = torch.randn(B, sum(h * w for h, w in SHAPES), C, generator=g).to(dev).requires_grad_(True)
    R = torch.randn(mem.shape, generator=g).to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    assert net.training_tokens_supported(mem, SHAPES)

    def tokens():
        out = net.forward_tokens(mem, SHAPES)
        return out, torch.autograd.grad((out * R).sum(), [mem] + params)

    def nchw():  # the differentiable split -> NCHW -> forward() -> concatenate round trip of SalienceTransformer.forward
        maps = [m.transpose(1, 2).reshape(B, C, h, w) for m, (h, w) in zip(mem.split([h * w for h, w in SHAPES], 1), SHAPES)]
        out = torch.cat([f.flatten(2).transpose(1, 2) for f in net(OrderedDict(enumerate(maps))).values()], 1).contiguous()
        return out, torch.autograd.grad((out * R).sum(), [mem] + params)

    arms = {"forward_tokens": (tokens, None), "nchw_cudnn_fp32": (nchw, False), "nchw_cudnn_tf32": (nchw, True)}
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False

    # float64 reference: forward() of a float64 twin from the same state
    net64 = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=4).to(dev).double().train()
    net64.load_state_dict(net.state_dict())
    m64 = mem.detach().double().requires_grad_(True)
    maps64 = [m.transpose(1, 2).reshape(B, C, h, w) for m, (h, w) in
              zip(m64.split([h * w for h, w in SHAPES], 1), SHAPES)]
    out64 = torch.cat([f.flatten(2).transpose(1, 2) for f in net64(OrderedDict(enumerate(maps64))).values()], 1)
    g64 = torch.autograd.grad((out64 * R.double()).sum(), [m64] + list(net64.parameters()))
    out64 = out64.detach()
    w64 = [g64[1 + i] for i, p in enumerate(params) if any(p is q for q in conv_w)]
    del net64, maps64, m64

    n_launch, errs, syncs, peak = {}, {}, {}, {}
    from torch.profiler import ProfilerActivity, profile
    for name, (fn, tf32) in arms.items():
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        n_launch[name] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                out, grads = fn()
            finally:
                torch.cuda.set_sync_debug_mode("default")
        syncs[name] = sum(1 for x in w if "synchroniz" in str(x.message).lower() and "prototype" not in str(x.message))
        torch.cuda.synchronize()
        peak[name] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        wg = [grads[1 + i] for i, p in enumerate(params) if any(p is q for q in conv_w)]
        out = out.detach()
        errs[name] = {"out": float((out.double() - out64).abs().max()),
                      "grad_memory": float((grads[0].double() - g64[0]).abs().max()),
                      "grad_conv_weights": max(float((x.double() - y).abs().max()) for x, y in zip(wg, w64)),
                      "grad_conv_weights_rel": max(float((x.double() - y).abs().max() / y.abs().max()) for x, y in zip(wg, w64))}
        del out, grads

    # the same steps replayed from CUDA graphs (captured after warm-up): device-bound, without the eager host overhead
    def graphed(fn):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            fn()
        return graph.replay

    for name, (fn, tf32) in list(arms.items()):
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        arms[name + "_graph"] = (graphed(fn), tf32)
        n_launch[name + "_graph"], syncs[name + "_graph"] = 1, 0
        errs[name + "_graph"], peak[name + "_graph"] = errs[name], None
    res = {k: [] for k in arms}
    for _ in range(a.rounds):
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            res[name].append(timed(fn, a.reps, flush))

    # profile breakdown of the token arm (a run of its own)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            tokens()
        torch.cuda.synchronize()
    share = defaultdict(float)
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            share[family(e.key)] += e.self_device_time_total
    total = sum(share.values()) or 1.0
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev

    out = {"card": card(), "shapes": SHAPES, "batch": B, "channels": C, "arms": {},
           "token_profile_share": {k: round(v / total, 3) for k, v in sorted(share.items(), key=lambda kv: -kv[1])},
           "token_profile_ms_per_step": round(total / 3 / 1000, 3)}
    for name in arms:
        out["arms"][name] = {"ms": [round(t, 3) for t in res[name]], "launches": n_launch[name], "host_syncs": syncs[name],
                             "peak_mib": peak[name], "max_abs_err_vs_fp64": errs[name]}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
