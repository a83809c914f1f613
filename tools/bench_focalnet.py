"""FocalNet-L backbone at the config-2 shapes (bs = 2, one 3 x 800 x 1344 padded batch, focalnet_large_lrf_fl4, return_indices
(1, 2, 3)): FocalNetBackbone.forward_tokens against the reference's op chain in torch with TF32 off for cuDNN and cuBLAS (fp32), with
torch's defaults (TF32 convolutions, fp32 matmuls), with TF32 on for both, and with TF32 on both and channels-last tensors.  Then
"images -> encoder memory": backbone + ChannelMapper + SalienceTransformer.forward_encoder (the bench.py model, 6 layers) in one
CUDA graph, against the TF32 torch backbone feeding the same mapper and encoder in one CUDA graph.

  python tools/bench_focalnet.py [--arch focalnet_large_lrf_fl4] [--reps 10] [--rounds 3] [--out FILE]

Every call is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating within
each round; "best" is the best round.  GFLOP: torch.utils.flop_counter on the torch module.  Launches: GPU kernels and memsets of
one call, counted with torch.profiler.  Errors: max |difference| / max |ref| per output against a float64 forward of the same
module.  Peak memory: torch.cuda.max_memory_allocated during one call, above what was allocated before it.  A separate profiled
call of forward_tokens splits GPU time by kernel kind.
"""
import argparse
import copy
import json
import os
import sys
from collections import OrderedDict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200 import synthetic  # noqa: E402
from salience_detr_b200.focalnet import FocalNet  # noqa: E402
from tools.bench_backbone import B, H, W, capture, card, gpu_events, peak_mb, timed  # noqa: E402


def set_tf32(conv, matmul):
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = conv, matmul


def kind(name):
    return ("gemm" if "gemm3x" in name else "scale" if "pow2" in name else "stem" if "stem" in name else
            "focal_level" if "focal_level" in name else "global_context" if "focal_global" in name else
            "modulate" if "modulate" in name else "conv" if "conv" in name else "layernorm" if "layernorm" in name else "other")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="focalnet_large_lrf_fl4")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_focalnet.py needs a GPU")
    dev = torch.device("cuda:0")
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    net = FocalNet(**pkg.FocalNetBackbone._config(a.arch, {}))
    weights = synthetic.focalnet_weights(net.state_dict(), 0)
    del net
    g = torch.Generator().manual_seed(0)
    x = torch.zeros(B, 3, H, W)
    x[0] = torch.randn(3, H, W, generator=g)
    x[1, :, :800, :1333] = torch.randn(3, 800, 1333, generator=g)  # the config's 800 x 1333 image padded to 1344
    x = x.to(dev)
    x_cl = x.contiguous(memory_format=torch.channels_last)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    from torch.utils.flop_counter import FlopCounterMode

    result = {"card": card(), "arch": a.arch, "batch": B, "image": [3, H, W], "return_indices": [1, 2, 3]}
    m = pkg.FocalNetBackbone(a.arch, weights=weights, return_indices=(1, 2, 3), freeze_indices=(0,)).to(dev).eval()
    m_cl = copy.deepcopy(m).to(memory_format=torch.channels_last)
    with torch.no_grad():
        with FlopCounterMode(display=False) as fc:
            m.forward_torch(x)
        gflop = fc.get_total_flops() / 1e9
        arms = {"tokens": (lambda: m.forward_tokens(x), None),
                "torch_fp32": (lambda: m.forward_torch(x), (False, False)),
                "torch_defaults": (lambda: m.forward_torch(x), (True, False)),
                "torch_tf32": (lambda: m.forward_torch(x), (True, True)),
                "torch_tf32_channels_last": (lambda: m_cl.forward_torch(x_cl), (True, True))}
        ref = copy.deepcopy(m).double()(x.double())
        info = {}
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                set_tf32(*tf32)
            for _ in range(3):
                out = fn()
            n0 = pkg.cabi.launch_count()
            fn()
            info[name] = {"library_launches": pkg.cabi.launch_count() - n0, "gpu_kernels": len(gpu_events(fn)),
                          "peak_mb": peak_mb(fn),
                          "rel_err_vs_fp64": {k: float((v.double() - ref[k]).abs().max() / ref[k].abs().max())
                                              for k, v in out.items()}}
            del out
        del ref
        res = {k: [] for k in arms}
        for _ in range(a.rounds):
            for name, (fn, tf32) in arms.items():
                if tf32 is not None:
                    set_tf32(*tf32)
                res[name].append(timed(fn, a.reps, flush))
        set_tf32(*prev)
    result.update({"gflop": round(gflop, 1), "launches_per_forward": m.launches_per_forward(), "arms": {}})
    for name in arms:
        best = min(res[name])
        result["arms"][name] = {"ms_rounds": [round(t, 3) for t in res[name]], "ms_best": round(best, 3),
                                "tflops_best": round(gflop / best, 1), **info[name]}
    for name in ("torch_fp32", "torch_defaults", "torch_tf32", "torch_tf32_channels_last"):
        result[f"speedup_tokens_vs_{name}"] = round(min(res[name]) / min(res["tokens"]), 3)

    # profiler split of one forward_tokens call by kernel kind
    with torch.no_grad():
        evs = [e for e in gpu_events(lambda: m.forward_tokens(x)) if "emset" not in e.name]
    split, calls = OrderedDict(), OrderedDict()
    for e in evs:
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        k = kind(e.name)
        split[k] = split.get(k, 0.0) + us
        calls[k] = calls.get(k, 0) + 1
    total = sum(split.values())
    result["profile"] = {k: {"calls": calls[k], "us": round(v, 1), "share": round(v / total, 3)} for k, v in split.items()}

    # images -> encoder memory in one CUDA graph
    mapper = pkg.ChannelMapper(m.num_channels, 256, 4).to(dev).eval()
    model = synthetic.build_model().to(dev).eval()
    model.attach_position_embedding(pkg.PositionEmbeddingSine(128, temperature=10000, normalize=True, offset=-0.5))
    _, masks_h, _ = synthetic.make_inputs("resnet50_800_1333_bs2", seed=0)
    masks = [mm.to(dev) for mm in masks_h]
    with torch.no_grad():
        plan = model.make_plan(masks)
        set_tf32(True, True)
        e2e = {"images_to_memory_tokens_graph": capture(lambda: model.forward_encoder(mapper(m(x)), masks, None, plan=plan)[0]),
               "images_to_memory_torch_tf32_graph": capture(lambda: model.forward_encoder(mapper(m.forward_torch(x)), masks, None,
                                                                                          plan=plan)[0])}
        res = {k: [] for k in e2e}
        for _ in range(a.rounds):
            for name, (graph, _) in e2e.items():
                res[name].append(timed(graph.replay, a.reps, flush))
        set_tf32(*prev)
    mem = {k: out for k, (_, out) in e2e.items()}
    result["e2e"] = {k: {"ms_rounds": [round(t, 3) for t in v], "ms_best": round(min(v), 3)} for k, v in res.items()}
    result["e2e"]["memory_max_abs_diff"] = float((mem["images_to_memory_tokens_graph"] -
                                                  mem["images_to_memory_torch_tf32_graph"]).abs().max())
    result["card_after"] = card()
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
