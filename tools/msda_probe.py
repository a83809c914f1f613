"""Where does the fused MSDA forward lose time?  Three conditions on the layer inputs captured from a real config-2 forward:
  cold    -- L2 flushed before every launch (value slice from HBM: the round-1 roofline definition)
  warm    -- the layer's value slice read once right before the launch (L2-resident, as after the per-layer value_proj GEMM)
  allhit  -- every query samples the SAME location (reference point 0.5, zero offsets): ~100 % L1 hits; the gap between
             this and `warm` is what L1 misses cost, i.e. the most a shared-memory/TMA-staged variant could win
Usage: python tools/msda_probe.py [option=value ...]   (options of sdetr_set_option)"""
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200.synthetic import build_model, make_inputs  # noqa: E402

dev = torch.device("cuda:0")
model = build_model().to(dev)
feats, masks, pos = make_inputs("resnet50_800_1333_bs2", seed=0, device=dev)
cabi = pkg.cabi
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
# variants: "name:opt=val,opt=val" ... (first = reference for the error column)
variants = [a for a in sys.argv[1:]] or ["default:"]
DEFAULTS = {"msda_tma": 0, "msda_warp_per_item": 0, "msda_threads": 256, "msda_chunk": 64, "msda_smem_broadcast": 1, "msda_min_blocks": 4}


def apply(spec):
    for k, v in DEFAULTS.items():
        cabi.set_option(k, v)
    name, _, opts = spec.partition(":")
    for kv in filter(None, opts.split(",")):
        k, v = kv.split("=")
        cabi.set_option(k, int(v))
    return name

calls = []
orig = cabi.msda_fused_forward


def spy(*a, **k):
    calls.append((list(a), k))
    return orig(*a, **k)


cabi.msda_fused_forward = spy
with torch.no_grad():
    plan = model.make_plan(masks)
    model.forward_encoder(feats, masks, pos, plan=plan, use_order=True)
cabi.msda_fused_forward = orig
torch.cuda.synchronize()
cabi.msda_set_host_shapes(plan.shapes_list)  # the TMA variant encodes its tensor maps on the host
b, nv = plan.mask_flat.shape
byts = [b * (4 * nv * 256 + nq * (12 * 128 + 4 * 256)) for nq in plan.layer_num_query]


def run(mode, reps=15):
    per = [[] for _ in calls]
    for _ in range(reps):
        for i, (a, k) in enumerate(calls):
            a = list(a)
            if mode == "allhit":
                a[6] = torch.full_like(a[6], 0.5)
                a[7] = torch.zeros_like(a[7])
            flush.zero_()
            if mode != "cold":
                a[0].sum()  # pulls the value slice into L2
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            orig(*a, **k)
            e1.record()
            torch.cuda.synchronize()
            per[i].append(e0.elapsed_time(e1) * 1000)
    return [statistics.median(x) for x in per]


print("value layout: token stride", calls[0][0][2], "floats")
print("variant            mode   | per-layer us | total us | GB/s algorithmic | clk per (query,head) per SM @1.965 GHz | max err vs first variant")
items = [b * nq * 8 for nq in plan.layer_num_query]
ref_out = None
for spec in variants:
    name = apply(spec)
    outs = [orig(*a, **k) for a, k in calls]
    torch.cuda.synchronize()
    if ref_out is None:
        ref_out = outs
    err = max((o - r).abs().max().item() for o, r in zip(outs, ref_out))
    for mode in ("cold", "warm", "allhit"):
        t = run(mode)
        cyc = sum(t) * 1e-6 * 1.98e9 * torch.cuda.get_device_properties(0).multi_processor_count / sum(items)  # at the H100 SXM max SM clock
        print(f"{name:18s} {mode:6s} | " + " ".join(f"{x:6.1f}" for x in t) + f" | {sum(t):7.1f} | {sum(byts) / sum(t) / 1e3:7.1f} | {cyc:6.1f} | {err:.1e}")
