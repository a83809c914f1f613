"""Denoising queries + denoising loss at config-2 shapes: this package's GenerateCDNQueries and compute_dn_loss against the
reference's op chain (GenerateCDNQueries.forward and DNDETRDetector.compute_dn_loss in torch, restated in oracle/denoising.py:
CPU index tensors, one calculate_loss per output, ``num_boxes`` read with ``.item()``).

Workload per call: bs = 2, C = 256, K = 91, 900 matching queries, 1 / 7 / 30 / 100 gts per image (G = 100 / 14 / 3 / 1
denoising groups): the generator's forward, the denoising loss of 6 decoder outputs over its 2*G*m queries (this package's
HybridSetCriterion in both arms, so the difference is the generator and the loss plumbing), then backward of the summed
losses plus a fixed linear functional of the label queries.  Protocol: CUDA events around synchronised calls, warm-up, three
alternating rounds; the card's name and power limit are read in the same run.  Prints one JSON line.

    python tools/bench_cdn.py [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import salience_detr_b200 as pkg  # noqa: E402
from oracle import denoising as odn  # noqa: E402
from oracle import set_criterion as osc  # noqa: E402
from tools.bench_criterion import card, sync_free, syncs_per_call, timed  # noqa: E402

BS, C, K, NQ, NUM_DN, DN_NUMS = 2, 256, 91, 900, 6, 100


def case(n_gt, seed=0):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(seed)
    tg = [{"boxes": osc.random_boxes(g, n_gt).to(dev), "labels": torch.randint(0, K, (n_gt,), generator=g).to(dev)}
          for _ in range(BS)]
    G = max(DN_NUMS * n_gt // n_gt ** 2, 1)
    pad = 2 * G * n_gt
    outs = [{"pred_logits": (torch.randn(BS, pad, K, generator=g) * 2 - 3).to(dev).requires_grad_(True),
             "pred_boxes": torch.stack([osc.random_boxes(g, pad) for _ in range(BS)]).to(dev).requires_grad_(True)}
            for _ in range(NUM_DN)]
    up = (torch.randn(BS, pad, C, generator=g) / pad).to(dev)
    dn_out = dict(outs[-1], aux_outputs=outs[:-1])
    return tg, dn_out, up, outs


def ours_step(gen, crit, tg, dn_out, up, leaves):
    for t in leaves:
        t.grad = None
    lq, bq, mask, G, m2 = gen([t["labels"] for t in tg], [t["boxes"] for t in tg])
    losses = pkg.compute_dn_loss(crit, {"denoising_groups": G, "max_gt_num_per_image": m2, "denoising_output": dn_out}, tg)
    (torch.stack(list(losses.values())).sum() + (lq * up).sum()).backward()


def ref_step(gen, crit, tg, dn_out, up, leaves):
    for t in leaves:
        t.grad = None
    lq, bq, mask, G, m2, _, _ = odn.cdn_queries(gen.label_encoder.weight, [t["labels"] for t in tg], [t["boxes"] for t in tg],
                                                gen.num_queries, gen.num_classes, gen.denoising_nums, gen.label_noise_prob,
                                                gen.box_noise_scale)
    nb = torch.as_tensor([float(sum(len(t["labels"]) for t in tg))], device=lq.device)
    nb = torch.clamp(nb, min=1).item()  # compute_dn_loss reads num_boxes on the host
    idx = []
    for t in tg:  # the per-image meshgrid of compute_dn_loss
        gi, ti = torch.meshgrid(torch.arange(G, device=lq.device), torch.arange(len(t["labels"]), device=lq.device),
                                indexing="ij")
        idx.append(((gi * m2 + ti).flatten(), ti.flatten()))
    losses = {}
    for j, o in enumerate([dn_out] + dn_out["aux_outputs"]):
        losses.update({f"{k}_{j}": v for k, v in crit.calculate_loss(o, tg, num_boxes=nb * G, indices=idx).items()})
    (torch.stack(list(losses.values())).sum() + (lq * up).sum()).backward()


def kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cdn needs a GPU")
    torch.manual_seed(0)
    gen = pkg.GenerateCDNQueries(NQ, K, C, DN_NUMS, 0.5, 1.0).cuda()
    c = osc.CONFIG
    crit = pkg.HybridSetCriterion(K, pkg.HungarianMatcher(c["cost_class"], c["cost_bbox"], c["cost_giou"], c["alpha"], c["gamma"]),
                                  {}, alpha=c["alpha"], gamma=c["gamma"])
    res = {"card": card(), "device": torch.cuda.get_device_name(),
           "workload": f"bs={BS} C={C} K={K} {NQ} queries: generator fwd + {NUM_DN} denoising outputs' loss + backward", "gt": {}}
    for n_gt in (1, 7, 30, 100):
        tg, dn_out, up, outs = case(n_gt)
        leaves = [gen.label_encoder.weight] + [t for o in outs for t in o.values()]
        ours = lambda: ours_step(gen, crit, tg, dn_out, up, leaves)  # noqa: E731
        ref = lambda: ref_step(gen, crit, tg, dn_out, up, leaves)  # noqa: E731
        for _ in range(3):
            ours(), ref()
        t_ours, t_ref = [], []
        for _ in range(3):  # alternating rounds
            t_ours.append(timed(ours, args.iters))
            t_ref.append(timed(ref, args.iters))
        gen_only = lambda: gen([t["labels"] for t in tg], [t["boxes"] for t in tg])[0].backward(up)  # noqa: E731
        t_gen = min(timed(gen_only, args.iters) for _ in range(3))
        gen_ref = lambda: odn.cdn_queries(gen.label_encoder.weight, [t["labels"] for t in tg], [t["boxes"] for t in tg], NQ, K,  # noqa: E731
                                          DN_NUMS, 0.5, 1.0)[0].backward(up)
        t_gen_ref = min(timed(gen_ref, args.iters) for _ in range(3))
        torch.cuda.synchronize()
        n0 = pkg.cabi.launch_count()
        ours()
        torch.cuda.synchronize()
        r = {"groups": max(DN_NUMS * n_gt // n_gt ** 2, 1), "ms_ours": round(min(t_ours), 3), "ms_ref": round(min(t_ref), 3),
             "ms_rounds_ours": [round(x, 3) for x in t_ours], "ms_rounds_ref": [round(x, 3) for x in t_ref],
             "ms_generator_fwd_bwd_ours": round(t_gen, 3),
             "ms_generator_fwd_bwd_ref": round(t_gen_ref, 3), "sdetr_launches_ours": pkg.cabi.launch_count() - n0,
             "gpu_kernels_and_copies_ours": kernels(ours), "gpu_kernels_and_copies_ref": kernels(ref),
             "sync_free_ours": sync_free(ours)}
        r["host_syncs_ours"], r["other_warnings_ours"] = syncs_per_call(ours)
        r["host_syncs_ref"], r["other_warnings_ref"] = syncs_per_call(ref)
        res["gt"][str(n_gt)] = r
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
