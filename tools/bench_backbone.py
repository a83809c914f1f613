"""ResNet-50 backbone at the config-2 shapes (bs = 2, one 3 x 800 x 1344 padded batch): ResNetBackbone.forward_tokens against
the reference's op chain on cuDNN with torch.backends.cudnn.allow_tf32 False (fp32) and True (torch's default, TF32), and TF32
with channels-last tensors; for return_indices (1, 2, 3) (the 4-scale config) and (0, 1, 2, 3) (the 5-scale config).  Then
"images -> encoder memory": backbone + ChannelMapper + SalienceTransformer.forward_encoder (the bench.py model, 6 layers) in one
CUDA graph, against the TF32 torch backbone feeding the same mapper and encoder in one CUDA graph.

  python tools/bench_backbone.py [--reps 10] [--rounds 3] [--out FILE]

Every call is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating within
each round; "best" is the best round.  GFLOP: torch.utils.flop_counter on the torch module (350.3 up to layer4).  Launches: GPU
kernels and memsets of one call, counted with torch.profiler.  Errors: max |difference| / max |ref| per output against a float64
forward of the same module.  Peak memory: torch.cuda.max_memory_allocated during one call, above what was allocated before it.
A separate profiled call of forward_tokens splits GPU time into convolutions (per shape), scale reductions, stem and pool.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
from collections import OrderedDict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200 import synthetic  # noqa: E402
from salience_detr_b200.backbone import ResNet  # noqa: E402

B, H, W = 2, 800, 1344


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


def gpu_events(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return round(peak / 2 ** 20, 1)


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    torch.cuda.synchronize()
    return graph, out


def conv_labels(m):
    """the convolutions of forward_tokens in launch order, as "layer<i>.<conv> <Cin>-><Cout> k<k>/s<s> <h>x<w>" labels"""
    out = []
    h, w = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    for li in range(max(m.return_indices) + 1):
        for blk in getattr(m, f"layer{li + 1}"):
            s = blk.conv2.stride[0]
            h2, w2 = (h - 1) // s + 1, (w - 1) // s + 1
            lab = lambda c, hh, ww: f"layer{li + 1}.{c} {getattr(blk, c).in_channels}->{getattr(blk, c).out_channels} " \
                                    f"k{getattr(blk, c).kernel_size[0]}/s{getattr(blk, c).stride[0]} out {hh}x{ww}"  # noqa: E731
            out += [lab("conv1", h, w), lab("conv2", h2, w2)]
            if blk.downsample is not None:
                ds = blk.downsample[0]
                out.append(f"layer{li + 1}.downsample {ds.in_channels}->{ds.out_channels} k1/s{ds.stride[0]} out {h2}x{w2}")
            out.append(lab("conv3", h2, w2))
            h, w = h2, w2
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_backbone.py needs a GPU")
    dev = torch.device("cuda:0")
    prev = torch.backends.cudnn.allow_tf32
    net = ResNet(**pkg.ResNetBackbone.model_arch["resnet50"], norm_layer=pkg.FrozenBatchNorm2d)
    weights = synthetic.resnet_weights({k: v.shape for k, v in net.state_dict().items() if not k.startswith("fc.")}, 0)
    g = torch.Generator().manual_seed(0)
    x = torch.zeros(B, 3, H, W)
    x[0] = torch.randn(3, H, W, generator=g)
    x[1, :, :800, :1333] = torch.randn(3, 800, 1333, generator=g)  # the config's 800 x 1333 image padded to 1344
    x = x.to(dev)
    x_cl = x.contiguous(memory_format=torch.channels_last)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from torch.utils.flop_counter import FlopCounterMode

    result = {"card": card(), "batch": B, "image": [3, H, W], "configs": {}}
    for ri in ((1, 2, 3), (0, 1, 2, 3)):
        m = pkg.ResNetBackbone("resnet50", weights=weights, return_indices=ri, freeze_indices=(0,),
                               norm_layer=pkg.FrozenBatchNorm2d).to(dev).eval()
        m_cl = copy.deepcopy(m).to(memory_format=torch.channels_last)
        with torch.no_grad():
            with FlopCounterMode(display=False) as fc:
                m.forward_torch(x)
            gflop = fc.get_total_flops() / 1e9
            arms = {"tokens": (lambda: m.forward_tokens(x), None),
                    "torch_cudnn_fp32": (lambda: m.forward_torch(x), False),
                    "torch_cudnn_tf32": (lambda: m.forward_torch(x), True),
                    "torch_cudnn_tf32_channels_last": (lambda: m_cl.forward_torch(x_cl), True)}
            ref = copy.deepcopy(m).double()(x.double())
            info = {}
            for name, (fn, tf32) in arms.items():
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                for _ in range(3):
                    out = fn()
                info[name] = {"launches": len(gpu_events(fn)), "peak_mb": peak_mb(fn),
                              "rel_err_vs_fp64": {k: float((v.double() - ref[k]).abs().max() / ref[k].abs().max())
                                                  for k, v in out.items()}}
                del out
            del ref
            res = {k: [] for k in arms}
            for _ in range(a.rounds):
                for name, (fn, tf32) in arms.items():
                    if tf32 is not None:
                        torch.backends.cudnn.allow_tf32 = tf32
                    res[name].append(timed(fn, a.reps, flush))
            torch.backends.cudnn.allow_tf32 = prev
        cfg = {"return_indices": list(ri), "gflop": round(gflop, 1), "library_launches": m.launches_per_forward(), "arms": {}}
        for name in arms:
            best = min(res[name])
            cfg["arms"][name] = {"ms_rounds": [round(t, 3) for t in res[name]], "ms_best": round(best, 3),
                                 "tflops_best": round(gflop / best, 1), **info[name]}
        cfg["speedup_tokens_vs_fp32"] = round(min(res["torch_cudnn_fp32"]) / min(res["tokens"]), 3)
        cfg["speedup_tokens_vs_tf32"] = round(min(res["torch_cudnn_tf32"]) / min(res["tokens"]), 3)
        result["configs"][str(ri)] = cfg

    # profiler split of one forward_tokens call (4-scale config)
    m = pkg.ResNetBackbone("resnet50", weights=weights, return_indices=(1, 2, 3), freeze_indices=(0,),
                           norm_layer=pkg.FrozenBatchNorm2d).to(dev).eval()
    with torch.no_grad():
        for _ in range(3):
            m.forward_tokens(x)
        evs = [e for e in gpu_events(lambda: m.forward_tokens(x)) if "Memset" not in e.name and "memset" not in e.name]
    split, convs = {"conv": 0.0, "scale": 0.0, "stem": 0.0, "pool": 0.0, "other": 0.0}, []
    for e in evs:
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        key = ("conv" if "conv_f16x3" in e.name else "scale" if "pow2" in e.name else "stem" if "stem" in e.name else
               "pool" if "maxpool" in e.name else "other")
        split[key] += us
        if key == "conv":
            convs.append(us)
    labels = conv_labels(m)
    per_shape = OrderedDict()
    for lab, us in zip(labels, convs):
        k = lab.split(" ", 1)[1]
        per_shape.setdefault(k, [0, 0.0])
        per_shape[k][0] += 1
        per_shape[k][1] += us
    result["profile_us"] = {k: round(v, 1) for k, v in split.items()}
    result["profile_conv_count"] = [len(convs), len(labels)]
    result["profile_conv_by_shape_us"] = {k: {"calls": n, "us": round(t, 1)} for k, (n, t) in per_shape.items()}

    # images -> encoder memory in one CUDA graph
    mapper = pkg.ChannelMapper([512, 1024, 2048], 256, 4).to(dev).eval()
    model = synthetic.build_model().to(dev).eval()
    model.attach_position_embedding(pkg.PositionEmbeddingSine(128, temperature=10000, normalize=True, offset=-0.5))
    _, masks_h, _ = synthetic.make_inputs("resnet50_800_1333_bs2", seed=0)
    masks = [mm.to(dev) for mm in masks_h]
    with torch.no_grad():
        plan = model.make_plan(masks)
        torch.backends.cudnn.allow_tf32 = True
        e2e = {"images_to_memory_tokens_graph": capture(lambda: model.forward_encoder(mapper(m(x)), masks, None, plan=plan)[0]),
               "images_to_memory_torch_tf32_graph": capture(lambda: model.forward_encoder(mapper(m.forward_torch(x)), masks, None,
                                                                                          plan=plan)[0])}
        res = {k: [] for k in e2e}
        for _ in range(a.rounds):
            for name, (graph, _) in e2e.items():
                res[name].append(timed(graph.replay, a.reps, flush))
        torch.backends.cudnn.allow_tf32 = prev
    mem = {k: out for k, (_, out) in e2e.items()}
    result["e2e"] = {k: {"ms_rounds": [round(t, 3) for t in v], "ms_best": round(min(v), 3)} for k, v in res.items()}
    result["e2e"]["memory_max_abs_diff"] = float((mem["images_to_memory_tokens_graph"] -
                                                  mem["images_to_memory_torch_tf32_graph"]).abs().max())
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
