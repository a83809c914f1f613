"""Detections on the GPU: a drop-in ``PostProcess`` whose sigmoid, top-k, box decode and filters are one launch.

``PostProcess`` mirrors the reference class (models/bricks/post_process.py:8-74): same constructor arguments and attributes,
same ``forward(outputs, target_sizes)`` -> ``[{"scores", "labels", "boxes"}]`` per image, with the reference's dtypes, shapes
and order.  The reference's chain of about a dozen torch launches (sigmoid, topk, div / mod, box conversion, gather, scale)
is ONE launch of ``sdetr_postprocess``:

* with both filters off there is no host synchronisation and the call can be captured in a CUDA graph; the per-image tensors
  are views of the (b, k) output buffers;
* with ``confidence_score > 0`` (optionally with ``nms_iou_threshold > 0``) the confidence filter and greedy NMS run in the
  same launch, and the b kept counts are read to the host once for the whole batch, instead of per-image boolean indexing and
  one ``torchvision.ops.nms`` call per image.

Differences from the reference:

* Ties of the sigmoid probability are ordered by the smaller flat (query * K + class) index, NaN first
  (``torch.sort(p, descending=True, stable=True)``); ``torch.topk`` leaves their order unspecified.  NMS visits the boxes in
  this order.
* Inputs must be CUDA tensors; ``pred_logits`` and ``pred_boxes`` float32, ``target_sizes`` int64, int32 or float32 (the
  reference would return float64 boxes for float64 sizes), ``select_box_nums_for_evaluation <= 4096``.  Anything else raises
  ``RuntimeError``.
"""
from __future__ import annotations

from typing import Dict, List

import torch
from torch import Tensor, nn

from . import cabi


class PostProcess(nn.Module):
    """models/bricks/post_process.py:8-74 on the GPU."""

    def __init__(self, select_box_nums_for_evaluation=100, nms_iou_threshold=-1, confidence_score=-1):
        super().__init__()
        self.select_box_nums_for_evaluation = select_box_nums_for_evaluation
        self.nms_iou_threshold = nms_iou_threshold
        self.confidence_score = confidence_score

    @torch.no_grad()
    def forward(self, outputs: Dict[str, Tensor], target_sizes: Tensor) -> List[Dict[str, Tensor]]:
        out_logits, out_bbox = outputs["pred_logits"], outputs["pred_boxes"]
        assert len(out_logits) == len(target_sizes)
        assert target_sizes.shape[1] == 2
        if self.nms_iou_threshold > 0 and not self.confidence_score > 0:
            # the reference builds the NMS masks from the confidence masks, which are None here (post_process.py:56)
            raise TypeError("'NoneType' object is not iterable: nms_iou_threshold > 0 needs confidence_score > 0")
        conf = self.confidence_score if self.confidence_score > 0 else -1.0
        iou = self.nms_iou_threshold if self.nms_iou_threshold > 0 else -1.0
        scores, labels, boxes, count = cabi.postprocess(out_logits, out_bbox, target_sizes, self.select_box_nums_for_evaluation,
                                                        conf, iou)
        if count is None:
            return [{"scores": s, "labels": l, "boxes": b} for s, l, b in zip(scores, labels, boxes)]
        kept = count.tolist()  # the one host synchronisation: the kept counts of the whole batch
        return [{"scores": s[:n], "labels": l[:n], "boxes": b[:n]} for s, l, b, n in zip(scores, labels, boxes, kept)]
