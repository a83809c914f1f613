"""TEST INFRASTRUCTURE ONLY -- plain-torch, device-agnostic restatement of the reference's GenerateCDNQueries.forward
(models/bricks/denoising.py:178-329, generate_query_masks :64-76, util/misc.py:31-35) and DNDETRDetector.compute_dn_loss
(models/detectors/base_detector.py:188-244), written from their semantics with the reference's op sequence.  The four random
draws are optional inputs: given, they replace the reference's draws; absent, they are drawn with the reference's calls in its
order.  Also the fixture cases of tests/golden/cdn_queries.npz (tools/make_cdn_golden.py)."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from oracle import set_criterion as osc

# tools/make_cdn_golden.py CASES: per case the gt counts, (num_queries, num_classes, label_embed_dim, denoising_nums,
# label_noise_prob, box_noise_scale) and the box style ("edges": boxes at the 0 / 1 borders and with zero size)
CASES = {
    "counts_3_7": dict(counts=(3, 7), cfg=(20, 11, 16, 100, 0.5, 1.0), boxes="random"),
    "empty_image": dict(counts=(0, 5), cfg=(20, 11, 16, 100, 0.5, 1.0), boxes="random"),
    "all_empty": dict(counts=(0, 0), cfg=(20, 11, 16, 100, 0.5, 1.0), boxes="random"),
    "m1_g100": dict(counts=(1, 1, 0), cfg=(10, 7, 8, 100, 0.5, 1.0), boxes="random"),
    "m120_g1": dict(counts=(120, 37), cfg=(30, 91, 8, 100, 0.5, 1.0), boxes="random"),
    "no_label_noise": dict(counts=(4, 2), cfg=(20, 11, 16, 100, 0.0, 1.0), boxes="random"),
    "no_box_noise": dict(counts=(4, 2), cfg=(20, 11, 16, 100, 0.5, 0.0), boxes="random"),
    "no_noise": dict(counts=(4, 2), cfg=(20, 11, 16, 100, 0.0, 0.0), boxes="random"),
    "edges": dict(counts=(8, 6), cfg=(20, 11, 16, 100, 0.5, 1.0), boxes="edges"),
}
INIT = dict(seed=3, cfg=(20, 11, 16, 100, 0.5, 1.0))  # the initial-weight check: manual_seed(seed), then construct


def case_inputs(name: str, seed: int):
    """-> (gt_labels_list, gt_boxes_list, cfg) of a fixture case, seeded, on the CPU."""
    c = CASES[name]
    g = torch.Generator().manual_seed(seed)
    K = c["cfg"][1]
    labels = [torch.randint(0, K, (n,), generator=g) for n in c["counts"]]
    boxes = [osc.random_boxes(g, n) for n in c["counts"]]
    if c["boxes"] == "edges":  # centres on the borders, zero / full sizes: reaches clamp(0, 1) and both eps clamps
        for b in boxes:
            n = b.shape[0]
            edge = torch.tensor([[0.0, 0.0, 0.0, 0.0], [1.0, 1.0, 0.0, 0.0], [0.5, 0.5, 1.0, 1.0], [0.0, 1.0, 0.2, 0.0],
                                 [1.0, 0.0, 0.0, 0.3], [0.9995, 0.0004, 0.001, 0.0008]])[:n]
            b[:edge.shape[0]] = edge
    return labels, boxes, c["cfg"]


def groups_of(counts: Sequence[int], denoising_nums: int) -> int:
    m = max(counts)
    return max(denoising_nums * m // max(m ** 2, 1), 1)


def inverse_sigmoid(x, eps: float = 1e-3, log=torch.log):
    x = x.clamp(min=0, max=1)
    x1 = x.clamp(min=eps)
    x2 = (1 - x).clamp(min=eps)
    return log(x1 / x2)


def cxcywh_to_xyxy(boxes):  # torchvision.ops.boxes._box_cxcywh_to_xyxy
    cx, cy, w, h = boxes.unbind(-1)
    return torch.stack((cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h), dim=-1)


def xyxy_to_cxcywh(boxes):  # torchvision.ops.boxes._box_xyxy_to_cxcywh
    x1, y1, x2, y2 = boxes.unbind(-1)
    return torch.stack(((x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1), dim=-1)


def query_mask(num_queries: int, groups: int, group_size: int, device) -> torch.Tensor:
    """generate_query_masks(group_size) with ``groups`` denoising groups"""
    d = group_size * groups
    mask = torch.zeros(d + num_queries, d + num_queries, device=device, dtype=torch.bool)
    mask[d:, :d] = True
    for i in range(groups):
        s, e = group_size * i, group_size * (i + 1)
        mask[s:e, :s] = True
        mask[s:e, e:d] = True
    return mask


def cdn_queries(weight, gt_labels_list: Sequence[torch.Tensor], gt_boxes_list: Sequence[torch.Tensor], num_queries: int,
                num_classes: int, denoising_nums: int, label_noise_prob: float, box_noise_scale: float,
                draws: Optional[Sequence[Optional[torch.Tensor]]] = None, log=torch.log):
    """GenerateCDNQueries.forward with label_encoder.weight ``weight`` -> (label_queries, box_queries, attn_mask, groups, 2m,
    draws used, noised labels (flat)).  ``log``: the logarithm of inverse_sigmoid (torch's CPU and CUDA log can differ in the
    last bit: passing CUDA's to a CPU run gives the CPU arithmetic with the GPU's log)."""
    counts = [x.numel() for x in gt_labels_list]
    m = max(counts)
    G = groups_of(counts, denoising_nums)
    gt_labels = torch.cat(list(gt_labels_list)).repeat(G * 2, 1).flatten()
    gt_boxes = torch.cat(list(gt_boxes_list)).repeat(G * 2, 1)
    device = gt_labels.device
    b = len(gt_labels_list)
    lr, li, bs, br = draws if draws is not None else (None,) * 4
    # apply_label_noise(labels, label_noise_prob * 0.5, num_classes)
    p = label_noise_prob * 0.5
    if p > 0:
        lr = torch.rand_like(gt_labels.float()) if draws is None else lr
        li = torch.randint_like(gt_labels, 0, num_classes) if draws is None else li
        noised_labels = torch.where(lr < p, li, gt_labels)
    else:
        noised_labels = gt_labels
    # apply_box_noise(boxes, box_noise_scale)
    boxes = gt_boxes
    if box_noise_scale > 0:
        S = len(boxes) // G // 2
        pos = torch.arange(S, dtype=torch.long, device=device).unsqueeze(0).repeat(G, 1)
        pos += torch.arange(G, dtype=torch.long, device=device).unsqueeze(1) * S * 2
        neg = pos.flatten() + S
        diff = torch.zeros_like(boxes)
        diff[:, :2] = boxes[:, 2:] / 2
        diff[:, 2:] = boxes[:, 2:] / 2
        bs = torch.randint_like(boxes, low=0, high=2, dtype=torch.float32) if draws is None else bs
        br = torch.rand_like(boxes) if draws is None else br
        rand_sign = bs * 2.0 - 1.0
        rand_part = br.clone()
        rand_part[neg] += 1.0
        rand_part *= rand_sign
        xyxy = cxcywh_to_xyxy(boxes)
        xyxy += torch.mul(rand_part, diff) * box_noise_scale
        boxes = xyxy_to_cxcywh(xyxy.clamp(min=0.0, max=1.0))
    boxes = inverse_sigmoid(boxes, log=log)
    emb = torch.nn.functional.embedding(noised_labels, weight)
    D = m * G * 2
    label_q = torch.zeros(b, D, weight.shape[1], device=device, dtype=weight.dtype)
    box_q = torch.zeros(b, D, 4, device=device)
    bi = torch.repeat_interleave(torch.arange(b), torch.tensor(counts, dtype=torch.long)).repeat(G * 2, 1).flatten()
    vi = torch.cat([torch.arange(n) for n in counts])
    vi = torch.cat([vi + m * i for i in range(G * 2)]).long()
    if len(bi):
        label_q = label_q.index_put((bi.to(device), vi.to(device)), emb)
        box_q[(bi.to(device), vi.to(device))] = boxes
    mask = query_mask(num_queries, G, 2 * m, device)
    return label_q, box_q, mask, G, 2 * m, (lr, li, bs, br), noised_labels


def dn_loss(dn_metas: Dict, targets: List[Dict], alpha=0.25, gamma=2.0) -> Dict[str, torch.Tensor]:
    """DNDETRDetector.compute_dn_loss with the oracle's calculate_loss: one call per denoising output and ``num_boxes`` read
    on the host with ``.item()``, as the reference does."""
    if "denoising_output" not in dn_metas:
        return {}
    out, G, max_gt = dn_metas["denoising_output"], dn_metas["denoising_groups"], dn_metas["max_gt_num_per_image"]
    device = out["pred_logits"].device
    nb = torch.as_tensor([sum(len(t["labels"]) for t in targets)], dtype=torch.float, device=device)
    nb = torch.clamp(nb, min=1).item()
    idx = []
    for t in targets:
        n = len(t["labels"])
        if n:
            gi, ti = torch.meshgrid(torch.arange(G, device=device), torch.arange(n, device=device), indexing="ij")
            idx.append(((gi * max_gt + ti).flatten(), ti.flatten()))
        else:
            idx.append((torch.tensor([], dtype=torch.long, device=device),) * 2)
    losses = {}
    for j, o in enumerate([out] + list(out.get("aux_outputs", []))):
        suf = "_dn" if j == 0 else f"_dn_{j - 1}"
        for k, v in osc.calculate_loss(o["pred_logits"], o["pred_boxes"], targets, nb * G, idx, alpha, gamma).items():
            losses[k + suf] = v
    return losses
