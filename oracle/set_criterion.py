"""TEST INFRASTRUCTURE ONLY -- plain torch (+ scipy) restatement of the reference's HungarianMatcher and HybridSetCriterion
(models/matcher/hungarian_matcher.py:7-91, models/bricks/set_criterion.py:14-212, models/bricks/losses.py:15-21), written
from their semantics.  ``dtype`` selects the arithmetic (float64 for gradient references).  Also: the seeded synthetic
inputs of the set-criterion fixtures (tests/golden/set_criterion_*.npz, tools/make_set_criterion_golden.py)."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

KEYS = ("loss_class", "loss_bbox", "loss_giou")
CONFIG = dict(cost_class=2.0, cost_bbox=5.0, cost_giou=2.0, alpha=0.25, gamma=2.0)  # configs/salience_detr/*


def xyxy(b):
    cx, cy, w, h = b.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)


def _inter_union_enclose(a, b):
    """Elementwise over broadcast xyxy boxes a, b: (inter, union, enclosing area); torch.max / torch.min / clamp as in
    torchvision's box ops, so autograd's tie conventions are the reference's."""
    area1 = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
    area2 = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    lt = torch.max(a[..., :2], b[..., :2])
    rb = torch.min(a[..., 2:], b[..., 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = area1 + area2 - inter
    lti = torch.min(a[..., :2], b[..., :2])
    rbi = torch.max(a[..., 2:], b[..., 2:])
    whi = (rbi - lti).clamp(min=0)
    return inter, union, whi[..., 0] * whi[..., 1]


def iou_giou(a, b):
    inter, union, enc = _inter_union_enclose(a, b)
    iou = inter / union
    return iou, iou - (enc - union) / enc


def cost_matrix(logits, boxes, gt_boxes, gt_labels, cost_class=2.0, cost_bbox=5.0, cost_giou=2.0, alpha=0.25, gamma=2.0):
    """(Q, K), (Q, 4), (n, 4), (n,) -> (Q, n) matching cost in the inputs' dtype."""
    prob = logits.sigmoid()
    neg = -(1 - alpha) * prob ** gamma * (1 - prob + 1e-6).log()
    pos = -alpha * (1 - prob) ** gamma * (prob + 1e-6).log()
    c_cls = pos[:, gt_labels] - neg[:, gt_labels]
    c_l1 = (boxes[:, None, :] - gt_boxes[None, :, :]).abs().sum(-1)
    _, giou = iou_giou(xyxy(boxes)[:, None, :], xyxy(gt_boxes)[None, :, :])
    return cost_bbox * c_l1 + cost_class * c_cls + cost_giou * -giou


def assign(cost) -> Tuple[torch.Tensor, torch.Tensor]:
    """scipy's exact assignment of a (Q, n) cost -> (src ascending, tgt) int64 CPU tensors."""
    from scipy.optimize import linear_sum_assignment

    r, c = linear_sum_assignment(cost.detach().cpu().numpy())
    return torch.as_tensor(r, dtype=torch.int64), torch.as_tensor(c, dtype=torch.int64)


def calculate_loss(logits, boxes, targets, num_boxes, indices, alpha=0.25, gamma=2.0) -> Dict[str, torch.Tensor]:
    """HybridSetCriterion.loss_labels + loss_boxes of one output: logits (b, Q, K), boxes (b, Q, 4); indices per image."""
    b, Q, K = logits.shape
    dev = logits.device
    indices = [(s.to(dev), t.to(dev)) for s, t in indices]
    bi = torch.cat([torch.full_like(s, i) for i, (s, _) in enumerate(indices)])
    si = torch.cat([s for s, _ in indices])
    src_boxes = boxes[bi, si]
    tgt_boxes = torch.cat([t["boxes"][j] for t, (_, j) in zip(targets, indices)]).to(boxes.dtype)
    iou, giou = iou_giou(xyxy(src_boxes), xyxy(tgt_boxes))
    classes = torch.full((b, Q), K, dtype=torch.int64, device=dev)
    classes[bi, si] = torch.cat([t["labels"][j] for t, (_, j) in zip(targets, indices)]).to(torch.int64)
    onehot = F.one_hot(classes, K + 1)[..., :-1]
    score = torch.zeros(b, Q, dtype=logits.dtype, device=dev)
    score[bi, si] = iou.detach()
    prob = logits.sigmoid().detach()
    t = onehot * score.unsqueeze(-1)
    w = (1 - alpha) * prob.pow(gamma) * (1 - onehot) + t
    lc = F.binary_cross_entropy_with_logits(logits, t, weight=w, reduction="none")
    return {"loss_class": (lc.sum(1) / max(Q, 1)).sum() / num_boxes * Q,
            "loss_bbox": F.l1_loss(src_boxes, tgt_boxes, reduction="none").sum() / num_boxes,
            "loss_giou": (1 - giou).sum() / num_boxes}


def num_boxes_of(targets) -> float:
    return max(float(sum(len(t["labels"]) for t in targets)), 1.0)


def match_output(logits, boxes, targets, cfg=CONFIG):
    return [assign(cost_matrix(lg, bx, t["boxes"].to(lg.dtype), t["labels"], cfg["cost_class"], cfg["cost_bbox"],
                               cfg["cost_giou"], cfg["alpha"], cfg["gamma"]))
            for lg, bx, t in zip(logits, boxes, targets)]


def criterion(outputs: Dict, targets: List[Dict], two_stage_binary_cls=False, cfg=CONFIG, indices: Optional[Dict] = None):
    """HybridSetCriterion.forward -> (losses, indices per suffix).  ``indices`` given: skip the matcher (same keys)."""
    nb = num_boxes_of(targets)
    items = [("", outputs, targets)]
    items += [(f"_{i}", a, targets) for i, a in enumerate(outputs.get("aux_outputs", []))]
    if "enc_outputs" in outputs:
        bt = [dict(t, labels=torch.zeros_like(t["labels"])) if two_stage_binary_cls else t for t in targets]
        items.append(("_enc", outputs["enc_outputs"], bt))
    losses, used = {}, {}
    for suf, out, tg in items:
        ind = indices[suf] if indices is not None else match_output(out["pred_logits"], out["pred_boxes"], tg, cfg)
        used[suf] = ind
        for k, v in calculate_loss(out["pred_logits"], out["pred_boxes"], tg, nb, ind, cfg["alpha"], cfg["gamma"]).items():
            losses[k + suf] = v
    return losses, used


# ---- seeded inputs of the fixtures -----------------------------------------------------------------------------------------
def random_boxes(g, n, dtype=torch.float32):
    c = torch.rand(n, 2, generator=g, dtype=torch.float64) * 0.8 + 0.1
    wh = torch.rand(n, 2, generator=g, dtype=torch.float64) * 0.3 + 0.02
    return torch.cat([c, wh], -1).to(dtype)


def synthetic_case(seed: int, bs: int, Q: int, K: int, gt_counts: Sequence[int], num_aux: int, enc_q: Optional[int],
                   dn_queries: int = 0, tie: bool = False):
    """-> (outputs, targets, dn_output or None) in float32.  Outputs: main + ``num_aux`` aux_outputs (+ enc_outputs with
    ``enc_q`` queries).  ``tie``: the main output's query 0 of the first non-empty image equals its gt 0 exactly."""
    g = torch.Generator().manual_seed(seed)
    targets = [{"boxes": random_boxes(g, n), "labels": torch.randint(0, K, (n,), generator=g)} for n in gt_counts]

    def out(q):
        return {"pred_logits": (torch.randn(bs, q, K, generator=g) * 2 - 3).float(),
                "pred_boxes": torch.stack([random_boxes(g, q) for _ in range(bs)])}

    main = out(Q)
    outputs = dict(main)
    outputs["aux_outputs"] = [out(Q) for _ in range(num_aux)]
    if enc_q:
        outputs["enc_outputs"] = out(enc_q)
    if tie:
        i = next(k for k, n in enumerate(gt_counts) if n)
        outputs["pred_boxes"][i, 0] = targets[i]["boxes"][0]
        outputs["pred_logits"][i, 0, targets[i]["labels"][0]] = 4.0
    dn = out(dn_queries) if dn_queries else None
    return outputs, targets, dn


def dn_indices(targets, groups: int, max_gt: int):
    """DNDETRDetector.compute_dn_loss's indices (base_detector.py:205-218), on the CPU."""
    idx = []
    for t in targets:
        n = len(t["labels"])
        if n:
            gi, ti = torch.meshgrid(torch.arange(groups), torch.arange(n), indexing="ij")
            idx.append(((gi * max_gt + ti).flatten(), ti.flatten()))
        else:
            idx.append((torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64)))
    return idx


def flat_outputs(outputs) -> List[Tuple[str, Dict]]:
    items = [("", outputs)] + [(f"_{i}", a) for i, a in enumerate(outputs.get("aux_outputs", []))]
    if "enc_outputs" in outputs:
        items.append(("_enc", outputs["enc_outputs"]))
    return items


def to_dtype(outputs, dtype, requires_grad=False):
    """Copy of ``outputs`` in ``dtype``, leaves with requires_grad."""
    def leaf(t):
        return t.detach().to(dtype).requires_grad_(requires_grad)
    new = {"pred_logits": leaf(outputs["pred_logits"]), "pred_boxes": leaf(outputs["pred_boxes"])}
    if "aux_outputs" in outputs:
        new["aux_outputs"] = [{k: leaf(v) for k, v in a.items()} for a in outputs["aux_outputs"]]
    if "enc_outputs" in outputs:
        new["enc_outputs"] = {k: leaf(v) for k, v in outputs["enc_outputs"].items()}
    return new


def same_assignment_fp32_fp64(outputs, targets, two_stage_binary_cls=False) -> bool:
    """True when scipy's assignment of every problem is the same for the fp32 and the fp64 cost (fixture seeds must pass)."""
    for suf, out in flat_outputs(outputs):
        tg = targets
        if suf == "_enc" and two_stage_binary_cls:
            tg = [dict(t, labels=torch.zeros_like(t["labels"])) for t in targets]
        a = match_output(out["pred_logits"], out["pred_boxes"], tg)
        b = match_output(out["pred_logits"].double(), out["pred_boxes"].double(), tg)
        if any(not (torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])) for x, y in zip(a, b)):
            return False
    return True


def sample_positions(seed: int, shape, count: int, must: np.ndarray) -> np.ndarray:
    """Sorted unique flat positions: ``count`` seeded ones plus ``must``."""
    rng = np.random.default_rng(seed)
    pos = rng.choice(int(np.prod(shape)), size=count, replace=False)
    return np.unique(np.concatenate([pos, must.astype(np.int64)]))
