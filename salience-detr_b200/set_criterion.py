"""Detection loss of a Salience-DETR training step on the GPU, without a host round trip.

``HungarianMatcher`` and ``HybridSetCriterion`` mirror the reference classes (models/matcher/hungarian_matcher.py:7-91,
models/bricks/set_criterion.py:14-212): same constructor arguments, same ``forward`` / ``calculate_loss`` signatures, same
unweighted loss keys.  What differs is where the work runs:

* every (output, image) problem of a step is matched in ONE launch (``sdetr_set_match``: cost matrix + exact shortest
  augmenting path assignment, the optimum scipy's ``linear_sum_assignment`` finds) instead of one device-to-host copy and one
  scipy call per problem;
* the losses of every output come from ONE ``torch.autograd.Function`` (two launches forward, one backward per 128
  (output, image) problems, i.e. per call up to a batch of 18 with 7 outputs) that returns an (outputs, 3) tensor; the loss
  dict entries are views of it;
* ``num_boxes`` is never read on the host: it is a host sum of the target sizes, or, under ``torch.distributed``, an
  all-reduced device tensor that the kernels divide by.

So a step with the real loss can run under ``torch.cuda.set_sync_debug_mode("error")`` and be captured in a CUDA graph.

Differences from the reference:

* ``HungarianMatcher.forward`` returns its index tensors on the device (int64), not on the CPU.
* A non-finite cost (NaN / inf logits or boxes) makes scipy raise ``ValueError``.  The batched path cannot raise without a
  sync: the problem is flagged on the device, gets a defined fallback assignment, and every loss of its output is NaN, which
  the caller's finite-loss check catches.  The per-image ``HungarianMatcher.forward`` reads the flag and raises ``ValueError``
  like the reference.
* Where several assignments reach the same minimum cost (exactly tied costs), the matcher may return a different one from
  scipy's: both are optimal, but the solver breaks ties toward the lowest query index and scipy's search visits the
  queries in another order.  The result is still deterministic.
* ``mixed_match`` (Align-DETR) is not implemented.
* Inputs must be CUDA tensors; CPU inputs raise ``RuntimeError``.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed
from torch import Tensor, nn

from . import cabi


def _rows(t: Tensor, name: str, width: Optional[int] = None) -> Tensor:
    """A CUDA float32 (..., Q, width) tensor whose last dimension is contiguous (views of stacked outputs are read in place)."""
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be float32, got {t.dtype}")
    if width is not None and t.shape[-1] != width:
        raise RuntimeError(f"{name} must have {width} columns, got {tuple(t.shape)}")
    return t if t.stride(-1) == 1 else t.contiguous()


def _gt(target: Dict, binary: bool) -> Tuple[Tensor, Optional[Tensor]]:
    boxes, labels = target["boxes"], target["labels"]
    if not (boxes.is_cuda and labels.is_cuda):
        raise RuntimeError("target boxes and labels must be CUDA tensors")
    boxes = boxes.to(torch.float32).contiguous()
    return boxes, None if binary else labels.to(torch.int64).contiguous()


def pair_offsets(counts: Sequence[int]) -> List[int]:
    """Offsets of each problem's pairs in the packed index buffer (exclusive prefix sum of the gt counts)."""
    offs, tot = [], 0
    for n in counts:
        offs.append(tot)
        tot += int(n)
    return offs


def num_boxes_of(targets: Sequence[Dict], device=None):
    """The reference's normaliser ``clamp(sum(len(labels)) / world_size, min=1)``: a Python float with world size 1 (no
    ``.item()``), a one-element device tensor that stays on the device under an initialised ``torch.distributed``."""
    n = sum(len(t["labels"]) for t in targets)
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        nb = torch.full((1,), float(n), dtype=torch.float32, device=device)
        torch.distributed.all_reduce(nb)
        return torch.clamp(nb / torch.distributed.get_world_size(), min=1)
    return max(float(n), 1.0)


class HungarianMatcher(nn.Module):
    """models/matcher/hungarian_matcher.py:7-91 on the GPU.  ``forward`` matches one image; :meth:`match` matches a whole
    batch of (output, image) problems in one launch."""

    def __init__(self, cost_class: float = 1, cost_bbox: float = 1, cost_giou: float = 1, focal_alpha: float = 0.25,
                 focal_gamma: float = 2.0, mixed_match: bool = False):
        super().__init__()
        self.cost_class = cost_class
        self.cost_bbox = cost_bbox
        self.cost_giou = cost_giou
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"
        self.focal_alpha = focal_alpha
        self.focal_gamma = focal_gamma
        if mixed_match:
            raise NotImplementedError("mixed_match (Align-DETR's repeated-gt assignment) is not implemented: no Salience-DETR "
                                      "config uses it")
        self.mixed_match = mixed_match

    def match(self, problems: Sequence[Tuple[Tensor, Tensor, Tensor, Optional[Tensor]]]):
        """problems: (pred_logits (Q, K), pred_boxes (Q, 4), gt_boxes (n, 4), gt_labels (n,) int64 or None for all-zero labels).
        -> (list of (src, tgt) int64 device tensors, views of one packed buffer; status (len(problems),) int32, 1 where a cost
        was not finite)."""
        if not problems:
            return [], None
        dev = problems[0][0].device
        counts = [int(p[2].shape[0]) for p in problems]
        offs = pair_offsets(counts)
        pairs = torch.empty(2, max(sum(counts), 1), dtype=torch.int64, device=dev)
        status = torch.empty(len(problems), dtype=torch.int32, device=dev)
        K = problems[0][0].shape[-1]
        structs, keep = [], []
        for (logits, boxes, gt_boxes, gt_labels), n, o in zip(problems, counts, offs):
            logits, boxes = _rows(logits, "pred_logits", K), _rows(boxes, "pred_boxes", 4)
            if logits.shape[0] != boxes.shape[0]:
                raise RuntimeError(f"pred_logits has {logits.shape[0]} queries, pred_boxes {boxes.shape[0]}")
            keep += [logits, boxes]
            structs.append(cabi.SetProblem(
                logits=logits.data_ptr(), boxes=boxes.data_ptr(), gt_boxes=gt_boxes.data_ptr() if n else None,
                gt_labels=gt_labels.data_ptr() if gt_labels is not None and n else None,
                src=pairs[0, o:].data_ptr(), tgt=pairs[1, o:].data_ptr(), logit_stride=logits.stride(0),
                box_stride=boxes.stride(0), num_queries=logits.shape[0], num_gt=n, num_pairs=n, output=0))
        for c in range(0, len(structs), cabi.SET_MAX_PROBLEMS):
            cabi.set_match(structs[c:c + cabi.SET_MAX_PROBLEMS], K, self.cost_class, self.cost_bbox, self.cost_giou,
                           self.focal_alpha, self.focal_gamma, status[c:c + cabi.SET_MAX_PROBLEMS])
        return [(pairs[0, o:o + n], pairs[1, o:o + n]) for o, n in zip(offs, counts)], status

    @torch.no_grad()
    def forward(self, pred_boxes: Tensor, pred_logits: Tensor, gt_boxes: Tensor, gt_labels: Tensor, gt_copy: int = 1):
        """One image: -> (src_ind, tgt_ind), int64 on the DEVICE (the reference returns CPU tensors).  Raises ``ValueError``
        on a non-finite cost like scipy and ``IndexError`` on a label outside [0, K) (both read the device: syncs)."""
        if not (gt_boxes.is_cuda and gt_labels.is_cuda):
            raise RuntimeError("gt_boxes and gt_labels must be CUDA tensors")
        if gt_labels.numel() and bool(((gt_labels < 0) | (gt_labels >= pred_logits.shape[-1])).any()):
            raise IndexError(f"gt label outside [0, {pred_logits.shape[-1]})")  # the reference's cost indexing raises here
        (ind,), status = self.match([(pred_logits, pred_boxes, gt_boxes.to(torch.float32).contiguous(),
                                      gt_labels.to(torch.int64).contiguous())])
        if bool(status[0]):
            raise ValueError("matrix contains invalid numeric entries")
        return ind


def _output_chunks(images_per_output: Sequence[int]) -> List[Tuple[int, int, int, int]]:
    """Consecutive whole outputs grouped into (first output, end output, first problem, end problem) chunks of at most
    cabi.SET_MAX_PROBLEMS problems each: a loss call sums every problem of an output, so an output never spans two calls."""
    chunks, o0, p0, p = [], 0, 0, 0
    for o, n in enumerate(images_per_output):
        if n > cabi.SET_MAX_PROBLEMS:
            raise RuntimeError(f"an output of {n} images exceeds the {cabi.SET_MAX_PROBLEMS} problems of one loss call")
        if p + n - p0 > cabi.SET_MAX_PROBLEMS:
            chunks.append((o0, o, p0, p))
            o0, p0 = o, p
        p += n
    if p > p0 or not chunks:
        chunks.append((o0, len(images_per_output), p0, p))
    return chunks


class _SetLoss(torch.autograd.Function):
    """(loss_class, loss_bbox, loss_giou) of several outputs from their matched pairs; -> (outputs, 3)."""

    @staticmethod
    def forward(ctx, spec, *preds):
        # spec: (per-output list of per-image (gt_boxes, gt_labels|None, src, tgt)), num_boxes, alpha, gamma, status
        per_output, num_boxes, alpha, gamma, status = spec
        logits_list, boxes_list = preds[0::2], preds[1::2]
        K = logits_list[0].shape[-1]
        chunks = _output_chunks([len(images) for images in per_output])
        first_output = {o: o0 for o0, o1, _, _ in chunks for o in range(o0, o1)}
        structs, keep = [], []
        for o, (logits, boxes, images) in enumerate(zip(logits_list, boxes_list, per_output)):
            logits, boxes = _rows(logits, "pred_logits", K), _rows(boxes, "pred_boxes", 4)
            keep += [logits, boxes]  # the kernels read these; copies made by _rows live as long as the pointers
            for i, (gtb, gtl, src, tgt) in enumerate(images):
                n = int(src.shape[0])
                structs.append(cabi.SetProblem(
                    logits=logits[i].data_ptr(), boxes=boxes[i].data_ptr(), gt_boxes=gtb.data_ptr() if gtb.numel() else None,
                    gt_labels=gtl.data_ptr() if gtl is not None and gtl.numel() else None, src=src.data_ptr() if n else None,
                    tgt=tgt.data_ptr() if n else None, logit_stride=logits.stride(1), box_stride=boxes.stride(1),
                    num_queries=logits.shape[1], num_gt=int(gtb.shape[0]), num_pairs=n, output=o - first_output[o]))
        loss = torch.empty(len(logits_list), 3, device=logits_list[0].device, dtype=torch.float32)
        for o0, o1, p0, p1 in chunks:
            cabi.set_loss_forward(structs[p0:p1], o1 - o0, K, alpha, gamma, status[p0:p1] if status is not None else None,
                                  num_boxes, loss[o0:o1])
        # the backward re-reads the predictions: saving them makes an in-place change before it an autograd error
        ctx.save_for_backward(*preds)
        ctx.state = (structs, keep, chunks, K, alpha, gamma, status, num_boxes, spec)
        ctx.shapes = [(tuple(lg.shape), tuple(bx.shape)) for lg, bx in zip(logits_list, boxes_list)]
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        ctx.saved_tensors  # noqa: B018 -- raises if a prediction was modified in place after the forward
        structs, keep, chunks, K, alpha, gamma, status, num_boxes, _ = ctx.state
        dev = grad_loss.device
        grads, k = [], 0
        for o, (ls, bs) in enumerate(ctx.shapes):
            gl = torch.empty(ls, device=dev, dtype=torch.float32)
            gb = torch.empty(bs, device=dev, dtype=torch.float32)
            grads += [gl, gb]
            for i in range(ls[0]):
                structs[k].grad_logits, structs[k].grad_boxes = gl[i].data_ptr(), gb[i].data_ptr()
                k += 1
        grad_loss = grad_loss.contiguous()
        for o0, o1, p0, p1 in chunks:
            cabi.set_loss_backward(structs[p0:p1], o1 - o0, K, alpha, gamma, status[p0:p1] if status is not None else None,
                                   num_boxes, grad_loss[o0:o1])
        return (None, *grads)


def set_losses(outputs: Sequence[Dict], images: Sequence[Sequence[Tuple]], num_boxes, alpha: float, gamma: float,
               status: Optional[Tensor] = None) -> Tensor:
    """Losses of several outputs in one call.  outputs[o]: {"pred_logits": (b, Q, K), "pred_boxes": (b, Q, 4)};
    images[o][i]: (gt_boxes, gt_labels or None, src, tgt) of image i.  -> (len(outputs), 3) (class, bbox, giou)."""
    preds = []
    for out in outputs:
        preds += [out["pred_logits"], out["pred_boxes"]]
    if torch.is_tensor(num_boxes):
        num_boxes = num_boxes.reshape(1).to(torch.float32)
    return _SetLoss.apply((list(images), num_boxes, alpha, gamma, status), *preds)


_KEYS = ("loss_class", "loss_bbox", "loss_giou")


class HybridSetCriterion(nn.Module):
    """models/bricks/set_criterion.py:173-212 (HybridSetCriterion over SetCriterion) on the GPU: the varifocal class loss with
    IoU-valued targets, L1 and GIoU box losses.  Returns the reference's unweighted dict; the detector applies
    ``weight_dict``."""

    def __init__(self, num_classes: int, matcher: nn.Module, weight_dict: Dict, alpha: float = 0.25, gamma: float = 2.0,
                 two_stage_binary_cls=False):
        super().__init__()
        self.num_classes = num_classes
        self.matcher = matcher
        self.weight_dict = weight_dict
        self.alpha = alpha
        self.gamma = gamma
        self.two_stage_binary_cls = two_stage_binary_cls

    def _losses(self, outputs: List[Dict], targets, num_boxes, binary: Sequence[bool], indices=None) -> Tensor:
        gts = {b: [_gt(t, b) for t in targets] for b in set(binary)}
        status = None
        if indices is None:
            problems = [(out["pred_logits"][i], out["pred_boxes"][i], *gts[b][i])
                        for out, b in zip(outputs, binary) for i in range(len(targets))]
            flat, status = self.matcher.match(problems)
            indices = [flat[k * len(targets):(k + 1) * len(targets)] for k in range(len(outputs))]
        else:
            if not all(s.is_cuda and t.is_cuda for s, t in indices):
                raise RuntimeError("indices must be CUDA tensors")
            indices = [[(s.to(torch.int64).contiguous(), t.to(torch.int64).contiguous()) for s, t in indices]] * len(outputs)
        images = [[(*gts[b][i], *indices[k][i]) for i in range(len(targets))] for k, b in enumerate(binary)]
        return set_losses(outputs, images, num_boxes, self.alpha, self.gamma, status)

    def calculate_loss(self, outputs, targets, num_boxes, indices=None, **kwargs):
        """The reference signature (set_criterion.py:120-131): with ``indices`` (the denoising path) the matcher is skipped.
        ``num_boxes``: a Python number or a one-element device tensor."""
        loss = self._losses([outputs], targets, num_boxes, [False], indices if indices else None)
        return {k: loss[0, c] for c, k in enumerate(_KEYS)}

    def forward(self, outputs, targets):
        num_boxes = num_boxes_of(targets, next(iter(outputs.values())).device)
        outs = [{k: v for k, v in outputs.items() if k not in ("aux_outputs", "enc_outputs")}]
        suffixes, binary = [""], [False]
        for i, aux in enumerate(outputs.get("aux_outputs", [])):
            outs.append(aux)
            suffixes.append(f"_{i}")
            binary.append(False)
        if "enc_outputs" in outputs:
            outs.append(outputs["enc_outputs"])
            suffixes.append("_enc")
            binary.append(bool(self.two_stage_binary_cls))
        loss = self._losses(outs, targets, num_boxes, binary)
        return {k + s: loss[o, c] for o, s in enumerate(suffixes) for c, k in enumerate(_KEYS)}
