"""Contrastive denoising queries of a Salience-DETR training step on the GPU, without a host round trip.

``GenerateCDNQueries`` mirrors the reference class (models/bricks/denoising.py:8-76, 178-329): same constructor arguments and
attributes, same ``label_encoder`` (a detector checkpoint's ``denoising_generator.label_encoder.weight`` loads), same
initialisation in the same RNG order, same ``forward`` 5-tuple.  What differs is where the work runs:

* ``forward`` draws the reference's four random tensors with the reference's torch calls, in its order and shapes, on the gt
  device, so on that device and generator state the noise is bit-identical; everything after the draws -- label noise, box
  noise, ``inverse_sigmoid``, the embedding lookup, the scatter into padded slots and the attention mask -- is ONE launch
  (``sdetr_cdn_queries``) instead of ~50 torch ops plus two mask fills per group and pageable host-to-device index copies;
* the embedding backward is one launch (``sdetr_cdn_queries_backward``) that sums each class row in slot order without atomics,
  so it is bit-reproducible, with or without ``torch.use_deterministic_algorithms(True)``;
* gt counts come from ``numel()`` (host metadata): no synchronisation, and a step with fixed gt counts can be captured in a
  CUDA graph.

:func:`compute_dn_loss` mirrors ``DNDETRDetector.compute_dn_loss`` (models/detectors/base_detector.py:188-244): its indices
come from one launch (``sdetr_cdn_loss_indices``), every denoising output goes through ONE ``HybridSetCriterion._losses``
call, and ``num_boxes`` is never read on the host.

Differences from the reference:

* A gt label that is still outside ``[0, num_classes)`` after the label noise makes the reference's embedding lookup raise.
  The kernel cannot raise without a sync: that query's label row is NaN and ``GenerateCDNQueries.status[i]`` (int32, on the
  device) is 1 for its image, so the caller's finite-loss check catches it.  The row gets no gradient.
* Inputs must be CUDA tensors (boxes float32); CPU inputs raise ``RuntimeError``.  At most 128 images per call.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
from torch import Tensor, nn

from . import cabi
from .set_criterion import _KEYS, num_boxes_of


class _CDNQueries(torch.autograd.Function):
    """label_encoder.weight -> (noised_label_queries, noised_box_queries, attn_mask, status); only the label queries carry a
    gradient."""

    @staticmethod
    def forward(ctx, spec, weight):
        labels, boxes, draws, K, C, threshold, scale, num_queries, groups, max_gt = spec
        label_q, box_q, noised, mask, status = cabi.cdn_queries(labels, boxes, draws, weight, K, C, threshold, scale,
                                                                num_queries, groups, max_gt)
        ctx.save_for_backward(noised)
        ctx.num_classes = K
        ctx.mark_non_differentiable(box_q, mask, status)
        return label_q, box_q, mask, status

    @staticmethod
    def backward(ctx, grad_label_q, _box, _mask, _status):
        (noised,) = ctx.saved_tensors
        return None, cabi.cdn_queries_backward(grad_label_q.contiguous(), noised, ctx.num_classes)


class GenerateCDNQueries(nn.Module):
    """models/bricks/denoising.py:178-329 (GenerateCDNQueries over GenerateDNQueries without indicator) on the GPU."""

    def __init__(self, num_queries: int = 300, num_classes: int = 80, label_embed_dim: int = 256, denoising_nums: int = 100,
                 label_noise_prob: float = 0.5, box_noise_scale: float = 1.0):
        super().__init__()
        # GenerateDNQueries.__init__(..., denoising_groups=1, with_indicator=False)
        self.num_queries = num_queries
        self.num_classes = num_classes
        self.label_embed_dim = label_embed_dim
        self.denoising_groups = 1
        self.label_noise_prob = label_noise_prob
        self.box_noise_scale = box_noise_scale
        self.with_indicator = False
        # the reference builds the embedding twice (the base class, then the subclass): the first one only consumes the
        # RNG, so that the weights equal the reference's under the same seed
        self.label_encoder = nn.Embedding(num_classes, label_embed_dim)
        self.denoising_nums = denoising_nums
        self.label_encoder = nn.Embedding(num_classes, label_embed_dim)
        self.status = None

    def draws(self, n: int, device) -> tuple:
        """The reference's random tensors over its repeated gt list of ``n`` entries, with its calls in its order
        (apply_label_noise, then apply_box_noise): (label_rand, label_randint, box_randint, box_rand), None where off."""
        lr = li = bs = br = None
        if self.label_noise_prob * 0.5 > 0:
            lr = torch.rand(n, device=device)
            li = torch.randint(0, self.num_classes, (n,), device=device)
        if self.box_noise_scale > 0:
            bs = torch.randint(0, 2, (n, 4), device=device, dtype=torch.float32)
            br = torch.rand(n, 4, device=device)
        return lr, li, bs, br

    def forward(self, gt_labels_list: Sequence[Tensor], gt_boxes_list: Sequence[Tensor]):
        """-> (noised_label_queries (b, 2Gm, C), noised_box_queries (b, 2Gm, 4), attn_mask (T, T) bool, G, 2m) with m the
        largest gt count, G = max(denoising_nums * m // m^2, 1), T = 2Gm + num_queries.  Sets ``denoising_groups`` and
        ``status``."""
        gt_nums_per_image = [x.numel() for x in gt_labels_list]
        max_gt_num_per_image = max(gt_nums_per_image)
        denoising_groups = self.denoising_nums * max_gt_num_per_image // max(max_gt_num_per_image**2, 1)
        self.denoising_groups = max(denoising_groups, 1)
        assert len(gt_labels_list) == len(gt_boxes_list)
        if not all(t.is_cuda for t in list(gt_labels_list) + list(gt_boxes_list)):
            raise RuntimeError("gt labels and boxes must be CUDA tensors")
        if any(b.dtype != torch.float32 for b in gt_boxes_list):
            raise RuntimeError("gt boxes must be float32")
        labels = [x.reshape(-1).to(torch.int64).contiguous() for x in gt_labels_list]
        boxes = [x.reshape(-1, 4).contiguous() for x in gt_boxes_list]
        if [b.shape[0] for b in boxes] != gt_nums_per_image:
            raise RuntimeError("every image needs one box per label")
        device = gt_labels_list[0].device
        draws = self.draws(2 * self.denoising_groups * sum(gt_nums_per_image), device)
        spec = (labels, boxes, draws, self.num_classes, self.label_embed_dim, self.label_noise_prob * 0.5, self.box_noise_scale,
                self.num_queries, self.denoising_groups, max_gt_num_per_image)
        label_q, box_q, attn_mask, self.status = _CDNQueries.apply(spec, self.label_encoder.weight)
        return label_q, box_q, attn_mask, self.denoising_groups, max_gt_num_per_image * 2


def compute_dn_loss(criterion, dn_metas: Dict, targets: List[Dict]) -> Dict[str, Tensor]:
    """DNDETRDetector.compute_dn_loss (base_detector.py:188-244) for this package's HybridSetCriterion: ``dn_metas`` is the
    dict ``dn_post_process`` fills ("denoising_output", "denoising_groups", "max_gt_num_per_image").  -> the reference's keys
    ``loss_{class,bbox,giou}_dn`` and ``..._dn_{i}`` per aux output."""
    if "denoising_output" not in dn_metas:
        return {}
    out, groups, max_gt = dn_metas["denoising_output"], dn_metas["denoising_groups"], dn_metas["max_gt_num_per_image"]
    device = out["pred_logits"].device
    num_boxes = num_boxes_of(targets, device) * groups
    pairs = cabi.cdn_loss_indices([len(t["labels"]) for t in targets], groups, max_gt, device)
    indices, o = [], 0
    for t in targets:
        n = groups * len(t["labels"])
        indices.append((pairs[0, o:o + n], pairs[1, o:o + n]))
        o += n
    outs = [out] + list(out.get("aux_outputs", []))
    loss = criterion._losses(outs, targets, num_boxes, [False] * len(outs), indices)
    suffixes = ["_dn"] + [f"_dn_{i}" for i in range(len(outs) - 1)]
    return {k + s: loss[j, c] for j, s in enumerate(suffixes) for c, k in enumerate(_KEYS)}
