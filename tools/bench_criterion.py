"""Detection loss forward + backward at config-2 shapes: this package's HybridSetCriterion against the reference's op chain
(torch on the GPU + scipy on the host per problem, restated in oracle/set_criterion.py).

Workload per call: bs = 2, Q = 900, K = 91, 6 decoder outputs + the encoder output (Q = 850) through the matcher, plus 6
denoising outputs through calculate_loss(indices=...), then backward of the summed losses.  gt counts per image: 7 (the COCO
mean), 30 and 100.  Protocol: CUDA events around synchronised calls, warm-up, three alternating rounds; the card's name and
power limit are read in the same run.  Prints one JSON line.

    python tools/bench_criterion.py [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import salience_detr_b200 as pkg  # noqa: E402
from oracle import set_criterion as osc  # noqa: E402

BS, Q, K, ENC_Q, NUM_DEC, NUM_DN = 2, 900, 91, 850, 6, 6


def case(n_gt, seed=0):
    groups = max(100 // n_gt, 1)
    outputs, targets, _ = osc.synthetic_case(seed, BS, Q, K, (n_gt,) * BS, NUM_DEC - 1, ENC_Q)
    g = torch.Generator().manual_seed(seed + 1)
    dn = [{"pred_logits": torch.randn(BS, groups * n_gt, K, generator=g) * 2 - 3,
           "pred_boxes": torch.stack([osc.random_boxes(g, groups * n_gt) for _ in range(BS)])} for _ in range(NUM_DN)]
    dev = torch.device("cuda")
    out = osc.to_dtype(outputs, torch.float32)
    leaves = []

    def mv(d):
        r = {k: v.to(dev).requires_grad_(True) for k, v in d.items() if torch.is_tensor(v)}
        leaves.extend(r.values())
        return r
    o = mv(out)
    o["aux_outputs"] = [mv(a) for a in out["aux_outputs"]]
    o["enc_outputs"] = mv(out["enc_outputs"])
    dn = [mv(d) for d in dn]
    tg = [{"boxes": t["boxes"].to(dev), "labels": t["labels"].to(dev)} for t in targets]
    ind = [(s.to(dev), t.to(dev)) for s, t in osc.dn_indices(targets, groups, n_gt)]
    return o, dn, tg, ind, groups, leaves


def ours_step(crit, o, dn, tg, ind, groups, leaves):
    for t in leaves:
        t.grad = None
    losses = crit(o, tg)
    nb = pkg.set_criterion.num_boxes_of(tg)
    for j, d in enumerate(dn):
        losses.update({f"{k}_dn_{j}": v for k, v in crit.calculate_loss(d, tg, nb * groups, indices=ind).items()})
    torch.stack(list(losses.values())).sum().backward()


def ref_step(o, dn, tg, ind, groups, leaves):
    for t in leaves:
        t.grad = None
    losses, _ = osc.criterion(o, tg)
    nb = osc.num_boxes_of(tg)
    for j, d in enumerate(dn):
        losses.update({f"{k}_dn_{j}": v for k, v in osc.calculate_loss(d["pred_logits"], d["pred_boxes"], tg, nb * groups,
                                                                   ind).items()})
    torch.stack(list(losses.values())).sum().backward()


def timed(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


SYNC_MESSAGE = "called a synchronizing CUDA operation"  # torch's set_sync_debug_mode warning


def syncs_per_call(fn):
    """-> (host synchronisations torch's sync debug mode reports in one call, texts of any other warning raised meanwhile)."""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
    msgs = [str(x.message) for x in w]
    return sum(SYNC_MESSAGE in m for m in msgs), sorted({m[:160] for m in msgs if SYNC_MESSAGE not in m})


def sync_free(fn) -> bool:
    """True when one call runs under set_sync_debug_mode("error") without raising."""
    torch.cuda.set_sync_debug_mode("error")
    try:
        fn()
        return True
    except RuntimeError:
        return False
    finally:
        torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_criterion needs a GPU")
    c = osc.CONFIG
    crit = pkg.HybridSetCriterion(K, pkg.HungarianMatcher(c["cost_class"], c["cost_bbox"], c["cost_giou"], c["alpha"], c["gamma"]),
                                  {}, alpha=c["alpha"], gamma=c["gamma"])
    res = {"card": card(), "device": torch.cuda.get_device_name(), "workload": f"bs={BS} Q={Q} K={K} {NUM_DEC} decoder + "
           f"encoder (Q={ENC_Q}) matched outputs + {NUM_DN} denoising outputs, forward + backward", "gt": {}}
    for n_gt in (7, 30, 100):
        o, dn, tg, ind, groups, leaves = case(n_gt)
        ours = lambda: ours_step(crit, o, dn, tg, ind, groups, leaves)  # noqa: E731
        ref = lambda: ref_step(o, dn, tg, ind, groups, leaves)  # noqa: E731
        for _ in range(3):
            ours(), ref()
        t_ours, t_ref = [], []
        for _ in range(3):  # alternating rounds
            t_ours.append(timed(ours, args.iters))
            t_ref.append(timed(ref, args.iters))
        problems = [(oo["pred_logits"][i], oo["pred_boxes"][i], t["boxes"], t["labels"])
                    for oo in [o] + o["aux_outputs"] + [o["enc_outputs"]] for i, t in enumerate(tg)]
        t_solver = min(timed(lambda: crit.matcher.match(problems), args.iters) for _ in range(3))
        n0 = pkg.cabi.launch_count()
        ours()
        torch.cuda.synchronize()
        launches = pkg.cabi.launch_count() - n0
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ours()
            torch.cuda.synchronize()
        kern_ours = sum(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ref()
            torch.cuda.synchronize()
        kern_ref = sum(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events())
        res["gt"][str(n_gt)] = {
            "ms_ours": round(min(t_ours), 3), "ms_ref": round(min(t_ref), 3), "ms_rounds_ours": [round(x, 3) for x in t_ours],
            "ms_rounds_ref": [round(x, 3) for x in t_ref], "ms_match_kernel_14_problems": round(t_solver, 3),
            "sdetr_launches_ours": launches, "gpu_kernels_and_copies_ours": kern_ours, "gpu_kernels_and_copies_ref": kern_ref,
            "sync_free_ours": sync_free(ours)}
        (res["gt"][str(n_gt)]["host_syncs_ours"], res["gt"][str(n_gt)]["other_warnings_ours"]) = syncs_per_call(ours)
        (res["gt"][str(n_gt)]["host_syncs_ref"], res["gt"][str(n_gt)]["other_warnings_ref"]) = syncs_per_call(ref)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
