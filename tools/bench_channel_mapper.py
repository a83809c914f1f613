"""ChannelMapper at the config-2 shapes (ResNet-50 maps 512@100x168, 1024@50x84, 2048@25x42, bs=2, out 256, plus the extra 3x3/s2
level to 13x21): forward_tokens from NCHW and from channels-last inputs, against the reference's NCHW op chain on cuDNN with
torch.backends.cudnn.allow_tf32 False (fp32) and True (torch's default, TF32); and "backbone maps -> encoder memory": the mapper
plus SalienceTransformer.forward_encoder (the bench.py model, 6 layers) captured in one CUDA graph, against the torch mapper (TF32,
torch's default) plus the same encoder in one CUDA graph.

  python tools/bench_channel_mapper.py [--reps 20] [--rounds 3] [--out FILE]

Every call is timed alone with CUDA events after a 256 MiB L2 flush, after warm-up; medians per round, the arms alternating within
each round.  GFLOP: torch.utils.flop_counter on the unfolded torch module at these shapes; TFLOP/s is that over the time.
Launches: GPU kernels and memsets of one call, counted with torch.profiler.  Errors: max |difference| from an fp64 torch forward
of the same module on the same maps.  "transpose_share": the three sdetr_token_map_transpose calls (NCHW -> token rows) timed
alone, over the NCHW forward_tokens time.
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
from tools import make_channel_mapper_golden as mcg  # noqa: E402

IN_CHANNELS, SHAPES, B, C = (512, 1024, 2048), [(100, 168), (50, 84), (25, 42)], 2, 256


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


def torch_forward(mapper, maps):
    """the reference's forward (channel_mapper.py:71-80) on the module's layers: cuDNN convolutions and GroupNorm in NCHW"""
    outs = [mapper.convs[i](maps[i]) for i in range(len(maps))]
    for i in range(len(maps), len(mapper.convs)):
        outs.append(mapper.convs[i](maps[-1] if i == len(maps) else outs[-1]))
    return outs


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_channel_mapper.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(mcg.MAPPER_SEED)
    mapper = mcg.perturb_affine(pkg.ChannelMapper(list(IN_CHANNELS), C, 4)).to(dev).eval()
    g = torch.Generator().manual_seed(0)
    nchw = [torch.randn(B, c, h, w, generator=g).to(dev) for c, (h, w) in zip(IN_CHANNELS, SHAPES)]
    cl = [x.contiguous(memory_format=torch.channels_last) for x in nchw]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    prev = torch.backends.cudnn.allow_tf32

    from salience_detr_b200.synthetic import build_model, make_inputs
    from torch.utils.flop_counter import FlopCounterMode

    model = build_model().to(dev).eval()
    model.attach_position_embedding(pkg.PositionEmbeddingSine(model.embed_dim // 2, temperature=10000, normalize=True, offset=-0.5))
    _, masks_h, _ = make_inputs("resnet50_800_1333_bs2", seed=0)
    masks = [m.to(dev) for m in masks_h]

    with torch.no_grad():
        plan = model.make_plan(masks)
        assert plan.shapes_list == SHAPES + [(13, 21)], plan.shapes_list
        with FlopCounterMode(display=False) as fc:
            torch_forward(mapper, nchw)
        gflop = fc.get_total_flops() / 1e9
        arms = {
            "tokens_nchw": (lambda: mapper.forward_tokens(nchw)[0], None),
            "tokens_channels_last": (lambda: mapper.forward_tokens(cl)[0], None),
            "nchw_transposes": (lambda: [pkg.cabi.maps_to_tokens([x]) for x in nchw], None),
            "torch_cudnn_fp32": (lambda: torch_forward(mapper, nchw), False),
            "torch_cudnn_tf32": (lambda: torch_forward(mapper, nchw), True),
        }
        torch.backends.cudnn.allow_tf32 = True  # torch's default: what an unmodified detector gets
        e2e = {"maps_to_memory_tokens_graph": capture(lambda: model.forward_encoder(mapper(OrderedDict(enumerate(nchw))), masks, None, plan=plan)[0]),
               "maps_to_memory_torch_tf32_graph": capture(lambda: model.forward_encoder(torch_forward(mapper, nchw), masks, None,
                                                                                          plan=plan)[0])}
        for name, (graph, _) in e2e.items():
            arms[name] = (graph.replay, None)
        n_launch, err = {}, {}
        for name, (fn, tf32) in arms.items():
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            for _ in range(3):
                fn()
            n_launch[name] = launches(fn)
        m64 = pkg.ChannelMapper(list(IN_CHANNELS), C, 4).to(dev).double().eval()
        m64.load_state_dict(mapper.state_dict())
        want = torch.cat([o.flatten(2).transpose(1, 2) for o in torch_forward(m64, [x.double() for x in nchw])], 1)
        for name in ("tokens_nchw", "tokens_channels_last", "torch_cudnn_fp32", "torch_cudnn_tf32"):
            fn, tf32 = arms[name]
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            got = fn()
            got = got if torch.is_tensor(got) else torch.cat([o.flatten(2).transpose(1, 2) for o in got], 1)
            err[name] = float((got.double() - want).abs().max())
        e2e_mem = {name: out.clone() for name, (_, out) in e2e.items()}
        res = {k: [] for k in arms}
        for _ in range(a.rounds):
            for name, (fn, tf32) in arms.items():
                if tf32 is not None:
                    torch.backends.cudnn.allow_tf32 = tf32
                res[name].append(timed(fn, a.reps, flush))
        torch.backends.cudnn.allow_tf32 = prev
    med = {k: statistics.median(v) for k, v in res.items()}
    out = {"card": card(), "shapes_in": [[c, h, w] for c, (h, w) in zip(IN_CHANNELS, SHAPES)], "shapes_out": plan.shapes_list,
           "batch": B, "channels": C, "gflop": round(gflop, 2),
           "mb_in": round(sum(x.numel() for x in nchw) * 4 / 1e6, 1), "mb_out": round(B * sum(h * w for h, w in plan.shapes_list) * C * 4 / 1e6, 1),
           "library_launches_per_forward_tokens": {"nchw": mapper.launches_per_forward(), "channels_last": mapper.launches_per_forward(0)},
           "transpose_share": [round(t / n, 3) for t, n in zip(res["nchw_transposes"], res["tokens_nchw"])],
           "e2e_memory_max_abs_diff_tokens_vs_torch_tf32": float((e2e_mem["maps_to_memory_tokens_graph"] -
                                                                  e2e_mem["maps_to_memory_torch_tf32_graph"]).abs().max()),
           "arms": {}}
    for name in arms:
        arm = {"ms": [round(t, 3) for t in res[name]], "launches": n_launch[name]}
        if name not in ("nchw_transposes",) and not name.startswith("maps_to_memory"):
            arm["tflops"] = [round(gflop / t, 1) for t in res[name]]
        if name in err:
            arm["max_abs_err_vs_fp64"] = err[name]
        out["arms"][name] = arm
    out["speedup_tokens_nchw_vs_tf32"] = round(med["torch_cudnn_tf32"] / med["tokens_nchw"], 3)
    out["speedup_tokens_nchw_vs_fp32"] = round(med["torch_cudnn_fp32"] / med["tokens_nchw"], 3)
    out["speedup_e2e"] = round(med["maps_to_memory_torch_tf32_graph"] / med["maps_to_memory_tokens_graph"], 3)
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
