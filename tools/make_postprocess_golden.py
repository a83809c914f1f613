"""TEST INFRASTRUCTURE ONLY -- golden fixture of PostProcess, made by running the UNMODIFIED reference on the CPU.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_postprocess_golden.py

  postprocess.npz   per case of CASES and per image i: ``<case>.<i>.scores`` / ``.labels`` / ``.boxes`` as the reference's
                    PostProcess (models/bricks/post_process.py) returns them, and ``seed``.

Inputs are not stored: ``case_inputs`` regenerates them from the seed, and the tests use the same function.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "postprocess.npz")
SEED = 70

# name -> (batch, Q, K, k, nms_iou_threshold, confidence_score, kind)
CASES = {
    "q900_k100": (2, 900, 91, 100, -1, -1, "plain"),
    "q900_k300": (2, 900, 91, 300, -1, -1, "plain"),
    "bs1": (1, 900, 91, 100, -1, -1, "plain"),
    "bs4": (4, 900, 91, 300, -1, -1, "plain"),
    "q300_c80": (2, 300, 80, 100, -1, -1, "plain"),
    "confidence": (2, 900, 91, 300, -1, 0.5, "plain"),
    "confidence_nms": (2, 900, 91, 300, 0.5, 0.5, "plain"),
    "saturated": (2, 40, 10, 390, -1, -1, "saturated"),  # the cut at k falls inside the tie group of the zeros
    "zero_width": (2, 900, 91, 300, 0.5, 0.5, "zero_width"),
}


def case_inputs(name: str, seed: int):
    """-> (outputs {"pred_logits" (b, Q, K), "pred_boxes" (b, Q, 4)}, target_sizes (b, 2) int64 (h, w) of ragged images)."""
    b, Q, K, _, _, _, kind = CASES[name]
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(b, Q, K, generator=g) * 1.5 - 4.5  # about 100 of the 81 900 scores above 0.5
    cxcy = torch.rand(b, Q, 2, generator=g) * 0.9 + 0.05
    wh = torch.rand(b, Q, 2, generator=g) * 0.4 + 0.02
    if kind == "saturated":
        # sigmoid exactly 1.0 (logit >= ~17) and exactly 0 (logit <= ~-104), +-inf and one NaN: ties at both ends
        q = torch.randint(0, Q, (b, 40), generator=g)
        c = torch.randint(0, K, (b, 40), generator=g)
        for i in range(b):
            logits[i, q[i, :20], c[i, :20]] = torch.rand(20, generator=g) * 60 + 20
            logits[i, q[i, 20:], c[i, 20:]] = -torch.rand(20, generator=g) * 60 - 110
            logits[i, q[i, 0], c[i, 0]] = float("inf")
            logits[i, q[i, 21], c[i, 21]] = float("-inf")
        logits[0, 5, 7] = float("nan")
    if kind == "zero_width":
        wh[:, ::3, 0] = 0.0  # every third query: a zero-width box (zero-area pairs give IoU NaN)
    sizes = torch.stack([torch.randint(300, 1334, (b,), generator=g), torch.randint(300, 1334, (b,), generator=g)], 1)
    return {"pred_logits": logits, "pred_boxes": torch.cat([cxcy, wh], -1)}, sizes


def load_reference():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "bricks", "post_process.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the reference")
    sys.path.insert(0, ref)
    from models.bricks.post_process import PostProcess
    return PostProcess


def main():
    Ref = load_reference()
    arrays = {"seed": np.array(SEED)}
    for ci, (name, (b, Q, K, k, nms, conf, _)) in enumerate(CASES.items()):
        outputs, sizes = case_inputs(name, SEED + ci)
        res = Ref(select_box_nums_for_evaluation=k, nms_iou_threshold=nms, confidence_score=conf)(outputs, sizes)
        assert len(res) == b
        for i, r in enumerate(res):
            for key in ("scores", "labels", "boxes"):
                arrays[f"{name}.{i}.{key}"] = r[key].numpy()
    np.savez_compressed(OUT, **arrays)
    print(OUT, "bytes", os.path.getsize(OUT))


if __name__ == "__main__":
    main()
