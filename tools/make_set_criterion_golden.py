"""Writes tests/golden/set_criterion_{small,c2}.npz from the UNMODIFIED reference HungarianMatcher / HybridSetCriterion
(models/matcher/hungarian_matcher.py, models/bricks/set_criterion.py) on the CPU.  Needs SDETR_REFERENCE_ROOT.

Inputs are not stored: they are regenerated from the seed by oracle.set_criterion.synthetic_case.  A seed is used only when
scipy's assignment of every problem is the same for the fp32 and the fp64 cost, so that a few ulps of difference between two
implementations of log / pow cannot legitimately flip a match.  Stored: matched indices (fp32 cost, as the reference trains),
every loss key and the gradients of their sum w.r.t. logits and boxes, all computed in float64.

    SDETR_REFERENCE_ROOT=/path/to/Salience-DETR python tools/make_set_criterion_golden.py
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import set_criterion as osc  # noqa: E402

CASES = {
    # a few outputs: main + one aux + the encoder output with binary targets; full fp64 gradients
    "small": dict(seed=100, bs=2, Q=300, K=20, gt_counts=(7, 30), num_aux=1, enc_q=300, binary=True, tie=False, dn=0,
                  full=True),
    # config-2 shapes: 6 decoder outputs + the encoder output (Q = 850), an empty image, a pred box equal to its gt, and the
    # denoising calculate_loss(indices=...) of 100 denoising queries (one group of max_gt = 100)
    "c2": dict(seed=200, bs=2, Q=900, K=91, gt_counts=(100, 0), num_aux=5, enc_q=850, binary=False, tie=True, dn=100,
               full=False),
}


def load_reference():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "bricks", "set_criterion.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the reference")
    sys.path.insert(0, ref)
    # set_criterion.py imports util.utils, whose real module imports accelerate: world size 1, no process group
    if "util" not in sys.modules:
        pkg = types.ModuleType("util")
        pkg.__path__ = [os.path.join(ref, "util")]
        sys.modules["util"] = pkg
    uu = types.ModuleType("util.utils")
    uu.get_world_size = lambda: 1
    uu.is_dist_avail_and_initialized = lambda: False
    sys.modules["util.utils"] = uu
    from models.bricks.set_criterion import HybridSetCriterion
    from models.matcher.hungarian_matcher import HungarianMatcher
    return HungarianMatcher, HybridSetCriterion


def ref_indices(matcher, outputs, targets, binary):
    out = {}
    for suf, o in osc.flat_outputs(outputs):
        tg = [dict(t, labels=torch.zeros_like(t["labels"])) for t in targets] if suf == "_enc" and binary else targets
        out[suf] = [matcher(b, lg, t["boxes"], t["labels"]) for b, lg, t in zip(o["pred_boxes"], o["pred_logits"], tg)]
    return out


def same_fp32_fp64(matcher, outputs, targets, binary):
    a = ref_indices(matcher, outputs, targets, binary)
    b = ref_indices(matcher, osc.to_dtype(outputs, torch.float64), [dict(t, boxes=t["boxes"].double()) for t in targets], binary)
    return all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for k in a for x, y in zip(a[k], b[k])), a


def make(name, cfg, Matcher, Criterion):
    cc = osc.CONFIG
    matcher = Matcher(cost_class=cc["cost_class"], cost_bbox=cc["cost_bbox"], cost_giou=cc["cost_giou"],
                      focal_alpha=cc["alpha"], focal_gamma=cc["gamma"])
    crit = Criterion(cfg["K"], matcher, {}, alpha=cc["alpha"], gamma=cc["gamma"], two_stage_binary_cls=cfg["binary"])
    seed = cfg["seed"]
    while True:
        outputs, targets, dn = osc.synthetic_case(seed, cfg["bs"], cfg["Q"], cfg["K"], cfg["gt_counts"], cfg["num_aux"],
                                                  cfg["enc_q"], cfg["dn"], cfg["tie"])
        ok, idx = same_fp32_fp64(matcher, outputs, targets, cfg["binary"])
        if ok:
            break
        seed += 1
    arrays = {"seed": np.array(seed)}
    for suf, ind in idx.items():
        for i, (s, t) in enumerate(ind):
            arrays[f"src{suf}_{i}"], arrays[f"tgt{suf}_{i}"] = s.numpy(), t.numpy()
    out64 = osc.to_dtype(outputs, torch.float64, requires_grad=True)
    tg64 = [dict(t, boxes=t["boxes"].double()) for t in targets]
    losses = crit(out64, tg64)
    sum(losses.values()).backward()
    for k, v in losses.items():
        arrays["loss." + k] = np.array(v.item())
    for suf, o in osc.flat_outputs(out64):
        gl = o["pred_logits"].grad.numpy()
        arrays[f"gb{suf}"] = o["pred_boxes"].grad.numpy()
        if cfg["full"]:
            arrays[f"gl{suf}"] = gl
        else:  # a seeded sample of positions that includes every matched (image, query, label) logit
            K, Q = gl.shape[2], gl.shape[1]
            tg = targets if not (suf == "_enc" and cfg["binary"]) else None
            must = [i * Q * K + s * K + (tg[i]["labels"][t] if tg is not None else 0)
                    for i, (ss, tt) in enumerate(idx[suf]) for s, t in zip(ss.tolist(), tt.tolist())]
            pos = osc.sample_positions(seed + len(suf), gl.shape, 2048, np.array(must, dtype=np.int64))
            arrays[f"gl_pos{suf}"], arrays[f"gl{suf}"] = pos, gl.reshape(-1)[pos]
    if dn is not None:
        dn64 = osc.to_dtype(dn, torch.float64, requires_grad=True)
        groups, max_gt = 1, max(cfg["gt_counts"])
        nb = osc.num_boxes_of(targets) * groups
        dl = crit.calculate_loss(dn64, tg64, num_boxes=nb, indices=osc.dn_indices(targets, groups, max_gt))
        sum(dl.values()).backward()
        for k, v in dl.items():
            arrays["dn." + k] = np.array(v.item())
        arrays["dn.gb"] = dn64["pred_boxes"].grad.numpy()
        arrays["dn.gl"] = dn64["pred_logits"].grad.numpy().astype(np.float64)
        arrays["dn.groups"], arrays["dn.max_gt"] = np.array(groups), np.array(max_gt)
    path = os.path.join(ROOT, "tests", "golden", f"set_criterion_{name}.npz")
    np.savez_compressed(path, **arrays)
    print(path, "seed", seed, "bytes", os.path.getsize(path))


def main():
    Matcher, Criterion = load_reference()
    for name in sys.argv[1:] or CASES:
        make(name, CASES[name], Matcher, Criterion)


if __name__ == "__main__":
    main()
