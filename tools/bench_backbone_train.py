"""ResNet-50 backbone training step at config 2 (bs 2, one 3x800x1344 padded batch, freeze_indices=(0,)): one forward +
backward of sum_k sum(out_k * R_k) for fixed random R_k, with forward_tokens under autograd (eager, and replayed from a CUDA
graph) against forward() on cuDNN fp32 (TF32 off), on cuDNN TF32, and on cuDNN TF32 with channels-last weights and input.
Run for return_indices=(1, 2, 3) (the shipped configs) and (0, 1, 2, 3) (the 5-scale ones).

  python tools/bench_backbone_train.py [--reps 10] [--rounds 3] [--out FILE]

Every step is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating
within each round.  Also per arm: TFLOP/s (the FLOPs torch.utils.flop_counter counts for forward() + backward, the same for
every arm), library launches (sdetr_launch_count) and GPU kernels and memsets (torch.profiler) per step, peak memory of a step,
and the worst max |err| / max |ref| over the trainable weights' gradients against forward() in float64.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200 import backbone as bbm, synthetic  # noqa: E402
from tools import make_backbone_golden as mbg  # noqa: E402

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


def images(dev):
    """the padded batch: image i of (H - 64 i) x (W - 96 i) pixels"""
    g = torch.Generator().manual_seed(0)
    x = torch.zeros(B, 3, H, W)
    for i in range(B):
        x[i, :, :H - 64 * i, :W - 96 * i] = torch.randn(3, H - 64 * i, W - 96 * i, generator=g)
    return x.to(dev)


def bench(return_indices, reps, rounds, dev, flush):
    net = bbm.ResNet(**pkg.ResNetBackbone.model_arch["resnet50"], norm_layer=pkg.FrozenBatchNorm2d)
    sd = synthetic.resnet_weights({k: list(v.shape) for k, v in net.state_dict().items() if not k.startswith("fc.")},
                                  mbg.WEIGHT_SEED)
    m = pkg.ResNetBackbone("resnet50", weights=sd, return_indices=return_indices, freeze_indices=(0,),
                           norm_layer=pkg.FrozenBatchNorm2d).to(dev)
    m_cl = copy.deepcopy(m).to(memory_format=torch.channels_last)
    x = images(dev)
    x_cl = x.contiguous(memory_format=torch.channels_last)
    assert m.training_tokens_supported(x)
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    with torch.no_grad():
        shapes = {k: v.shape for k, v in m.forward_tokens(x).items()}
    g = torch.Generator().manual_seed(1)
    R = {k: torch.randn(s, generator=g).to(dev) for k, s in shapes.items()}

    def step(mm, xx, tokens):
        params = [p for p in mm.parameters() if p.requires_grad]
        outs = mm.forward_tokens(xx) if tokens else mm(xx)
        return torch.autograd.grad(sum((v * R[k]).sum() for k, v in outs.items()), params)

    arms = {"tokens": (lambda: step(m, x, True), None), "cudnn_fp32": (lambda: step(m, x, False), False),
            "cudnn_tf32": (lambda: step(m, x, False), True), "cudnn_tf32_channels_last": (lambda: step(m_cl, x_cl, False), True)}

    # float64 reference and the FLOP count of forward() + backward
    m64 = copy.deepcopy(m).double()
    from torch.utils.flop_counter import FlopCounterMode
    with FlopCounterMode(display=False) as fc:
        outs = m64(x.double())
        g64 = torch.autograd.grad(sum((v * R[k].double()).sum() for k, v in outs.items()),
                                  [p for p in m64.parameters() if p.requires_grad])
    flops = fc.get_total_flops()
    del m64, outs

    from torch.profiler import ProfilerActivity, profile
    prev = torch.backends.cudnn.allow_tf32
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
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        n0 = pkg.cabi.launch_count()
        grads = fn()
        torch.cuda.synchronize()
        lib = pkg.cabi.launch_count() - n0
        peak = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
        rel = {n: float((a.double() - r).abs().max() / r.abs().max()) for n, a, r in zip(names, grads, g64)}
        worst = max(rel, key=rel.get)
        info[name] = {"library_launches": lib, "gpu_kernels": kernels, "peak_mib": peak,
                      "max_rel_err_weight_grads": rel[worst], "worst_param": worst}
        del grads

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

    arms["tokens_graph"] = (graphed(arms["tokens"][0]), None)
    info["tokens_graph"] = dict(info["tokens"], gpu_kernels=None, library_launches=None)
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            res[name].append(timed(fn, reps, flush))
    torch.backends.cudnn.allow_tf32 = prev
    out = {"return_indices": list(return_indices), "gflop_per_step": round(flops / 1e9, 1),
           "launches_per_training_step": m.launches_per_training_step(), "arms": {}}
    for name in arms:
        out["arms"][name] = dict(info[name], ms=[round(t, 3) for t in res[name]],
                                 tflops=round(flops / (statistics.median(res[name]) * 1e-3) / 1e12, 1))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {"card": card(), "batch": B, "image": [3, H, W],
           "configs": [bench(ri, a.reps, a.rounds, dev, flush) for ri in ((1, 2, 3), (0, 1, 2, 3))]}
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
