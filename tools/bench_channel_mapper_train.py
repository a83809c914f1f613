"""ChannelMapper training step at the config-2 shapes of ResNet-50 (512@100x168, 1024@50x84, 2048@25x42, bs=2, C=256, plus the
extra 3x3 / stride-2 level): one forward + backward of sum(out * R) for a fixed random R, once with inputs that require a
gradient (a trained backbone) and once with inputs that do not.

  python tools/bench_channel_mapper_train.py [--reps 10] [--rounds 3] [--out FILE]

Arms, alternating within each round, every step timed alone with CUDA events after a 256 MiB L2 flush:
  tokens / tokens_graph     forward_tokens under autograd on channels-last inputs, eager and replayed from a CUDA graph
  cudnn_fp32                forward() (the torch chain) on NCHW inputs, cuDNN with TF32 off
  cudnn_tf32                the same with TF32 on
  cudnn_tf32_cl             TF32 with channels-last inputs and weights
Per arm also: library launches (sdetr_launch_count), GPU kernels (torch.profiler), peak memory of a step, and max |error| /
max |ref| against forward() in float64 for the output, the input gradients, the convolution weight gradients and the GroupNorm
weight and bias gradients.  The chain arms put ResNet-50 forward_tokens training (freeze_indices=(0,), 2x3x800x1344) in front
of the mapper in one CUDA graph: the token mapper against the torch mapper (TF32 off and on).
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
from salience_detr_b200 import backbone as bbm, synthetic  # noqa: E402
from tools import make_backbone_golden as mbg  # noqa: E402
from tools import make_channel_mapper_golden as mcg  # noqa: E402

CIN = (512, 1024, 2048)
SHAPES = [(100, 168), (50, 84), (25, 42)]
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


def tokens_of(outs):
    return torch.cat([o.flatten(2).transpose(1, 2) for o in outs], 1)


def rel(a, ref):
    return float((a.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def mapper_bench(input_grad, reps, rounds, dev, flush):
    torch.manual_seed(5)
    m = mcg.perturb_affine(pkg.ChannelMapper(list(CIN), C, len(CIN) + 1)).to(dev).train()
    m_cl = copy.deepcopy(m).to(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(B, c, h, w, generator=g).to(dev) for c, (h, w) in zip(CIN, SHAPES)]
    nchw = OrderedDict((str(i), x.requires_grad_(input_grad)) for i, x in enumerate(xs))
    cl = OrderedDict((k, v.detach().contiguous(memory_format=torch.channels_last).requires_grad_(input_grad)) for k, v in nchw.items())
    nv = sum(h * w for h, w in SHAPES) + ((SHAPES[-1][0] - 1) // 2 + 1) * ((SHAPES[-1][1] - 1) // 2 + 1)
    R = torch.randn(B, nv, C, generator=g).to(dev)
    assert m.training_tokens_supported(cl)

    def step(mm, inputs, tokens):
        def fn():
            out = mm.forward_tokens(inputs)[0] if tokens else tokens_of(mm(inputs))
            xg = [x for x in inputs.values() if x.requires_grad]
            return out, torch.autograd.grad((out * R).sum(), xg + list(mm.parameters()))
        return fn

    arms = {"tokens": (step(m, cl, True), None), "cudnn_fp32": (step(m, nchw, False), False),
            "cudnn_tf32": (step(m, nchw, False), True), "cudnn_tf32_cl": (step(m_cl, cl, False), True)}
    # float64 reference
    m64 = copy.deepcopy(m).double()
    in64 = OrderedDict((k, v.detach().double().requires_grad_(input_grad)) for k, v in nchw.items())
    out64 = tokens_of(m64(in64))
    xg64 = [x for x in in64.values() if x.requires_grad]
    g64 = torch.autograd.grad((out64 * R.double()).sum(), xg64 + list(m64.parameters()))
    out64 = out64.detach()
    nx = len(xg64)
    names = [n for n, _ in m.named_parameters()]
    groups = {"input_grads": list(range(nx)),
              "conv_weight_grads": [nx + i for i, n in enumerate(names) if n.endswith(".0.weight")],
              "gn_weight_grads": [nx + i for i, n in enumerate(names) if n.endswith(".1.weight")],
              "gn_bias_grads": [nx + i for i, n in enumerate(names) if n.endswith(".1.bias")]}
    del m64, in64

    from torch.profiler import ProfilerActivity, profile
    info = {}
    for name, (fn, tf32) in arms.items():
        if tf32 is not None:
            torch.backends.cudnn.allow_tf32 = tf32
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        n0 = pkg.cabi.launch_count()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out, grads = fn()
        torch.cuda.synchronize()
        errs = {"out": rel(out.detach(), out64)}
        for k, idx in groups.items():
            if idx:
                errs[k] = max(rel(grads[i], g64[i]) for i in idx)
        info[name] = {"library_launches": pkg.cabi.launch_count() - n0, "gpu_kernels": kernels,
                      "peak_mib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1),
                      "max_err_over_max_ref_vs_fp64": {k: float(f"{v:.3e}") for k, v in errs.items()}}
        del out, grads
    torch.backends.cudnn.allow_tf32 = False
    arms["tokens_graph"] = (graphed(arms["tokens"][0]), None)
    info["tokens_graph"] = dict(info["tokens"], gpu_kernels=None)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            res[name].append(round(timed(fn, reps, flush), 3))
    for k in arms:
        info[k]["ms"] = res[k]
    return info


def chain_bench(reps, rounds, dev, flush):
    """images -> ResNet-50 forward_tokens training -> mapper -> sum(out * R) and its backward, one CUDA graph per arm"""
    net = bbm.ResNet(**pkg.ResNetBackbone.model_arch["resnet50"], norm_layer=pkg.FrozenBatchNorm2d)
    sd = synthetic.resnet_weights({k: list(v.shape) for k, v in net.state_dict().items() if not k.startswith("fc.")},
                                  mbg.WEIGHT_SEED)
    bb = pkg.ResNetBackbone("resnet50", weights=sd, return_indices=(1, 2, 3), freeze_indices=(0,),
                            norm_layer=pkg.FrozenBatchNorm2d).to(dev)
    torch.manual_seed(5)
    m = mcg.perturb_affine(pkg.ChannelMapper(list(CIN), C, len(CIN) + 1)).to(dev).train()
    g = torch.Generator().manual_seed(0)
    x = torch.zeros(B, 3, 800, 1344)
    for i in range(B):
        x[i, :, :800 - 64 * i, :1344 - 96 * i] = torch.randn(3, 800 - 64 * i, 1344 - 96 * i, generator=g)
    x = x.to(dev)
    params = [p for p in list(bb.parameters()) + list(m.parameters()) if p.requires_grad]
    nv = sum(h * w for h, w in SHAPES) + 13 * 21
    R = torch.randn(B, nv, C, generator=g).to(dev)

    def step(tokens):
        def fn():
            feats = bb.forward_tokens(x)
            out = m.forward_tokens(feats)[0] if tokens else tokens_of(m(feats))
            return torch.autograd.grad((out * R).sum(), params)
        return fn

    arms = {"chain_tokens_graph": (step(True), False), "chain_torch_mapper_fp32_graph": (step(False), False),
            "chain_torch_mapper_tf32_graph": (step(False), True)}
    for name, (fn, tf32) in list(arms.items()):
        torch.backends.cudnn.allow_tf32 = tf32
        arms[name] = (graphed(fn), tf32)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (fn, tf32) in arms.items():
            torch.backends.cudnn.allow_tf32 = tf32
            res[name].append(round(timed(fn, reps, flush), 3))
    return {k: {"ms": v} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        out = {"card": card(), "shapes": SHAPES, "in_channels": CIN, "batch": B, "channels": C,
               "inputs_require_grad": mapper_bench(True, a.reps, a.rounds, dev, flush),
               "inputs_without_grad": mapper_bench(False, a.reps, a.rounds, dev, flush),
               "chain": chain_bench(a.reps, a.rounds, dev, flush)}
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
