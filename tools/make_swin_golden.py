"""TEST INFRASTRUCTURE ONLY -- golden fixture of the Swin-L backbone, made by running the UNMODIFIED reference on the CPU.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_swin_golden.py

  swin_l_backbone.npz
    shapes_json        the reference feature extractor's state-dict keys and shapes (SwinTransformerBackbone("swin_l",
                       return_indices=(1, 2, 3), freeze_indices=(0,)))
    init_sums_json     per-tensor sums of the reference SwinTransformer's default initialisation (swin_l settings) under
                       torch.manual_seed(0), all keys but norm.* and head.*
    grad_json          requires_grad of every parameter after freeze_indices=(0,)
    num_channels_json  the extractor's num_channels
    image              (2, 3, 64, 100): image 0 full, image 1 a 56 x 84 image zero-padded into the batch
    out.features.3/5/7 the extractor's outputs on it with the synthetic.swin_weights(WEIGHT_SEED) weights, in eval mode

The image gives 16 x 25 tokens after the stem, so every stage pads to whole 7 x 7 windows (16 x 25 -> 21 x 28, 8 x 13 ->
14 x 14, ...), the first PatchMerging has an odd width, and the shift is on in stages 0-1 and disabled in stages 2-3 (the
window covers the padded map).  The weights are passed as a state dict, so nothing is downloaded.  The weights and the image
are regenerated from their seeds by weights() / image(), which the tests share.  The reference's own
SwinTransformerBackbone.__new__, load_checkpoint and load_state_dict run; only the third-party modules it imports and that are
not installed here are stubbed (make_backbone_golden's stubs).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.make_backbone_golden import _stub_missing_modules  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "swin_l_backbone.npz")
WEIGHT_SEED, IMAGE_SEED = 81, 82
RETURN_INDICES, FREEZE_INDICES = (1, 2, 3), (0,)
SWIN_L = dict(patch_size=(4, 4), embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window_size=(7, 7),
              stochastic_depth_prob=0.2)


def weights(state):
    """the fixture's weights for the network's state dict (synthetic.swin_weights)"""
    from salience_detr_b200 import synthetic

    return synthetic.swin_weights(state, WEIGHT_SEED)


def image():
    """(2, 3, 64, 100): a full image and a 56 x 84 one zero-padded to the batch size"""
    g = torch.Generator().manual_seed(IMAGE_SEED)
    x = torch.zeros(2, 3, 64, 100)
    x[0] = torch.randn(3, 64, 100, generator=g)
    x[1, :, :56, :84] = torch.randn(3, 56, 84, generator=g)
    return x


def main():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "backbones", "swin.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the original project")
    sys.path.insert(0, ref)
    _stub_missing_modules()
    from models.backbones.swin import SwinTransformer, SwinTransformerBackbone

    torch.manual_seed(0)
    init = SwinTransformer(**SWIN_L)
    keep = {k: v for k, v in init.state_dict().items() if not k.startswith(("norm.", "head."))}
    init_sums = {k: float(v.double().sum()) for k, v in keep.items()}
    w = weights(keep)
    del init

    net = SwinTransformerBackbone.__new__(SwinTransformerBackbone, "swin_l", weights=w, return_indices=RETURN_INDICES,
                                          freeze_indices=FREEZE_INDICES)
    extractor = net[0]
    grads = {k: p.requires_grad for k, p in extractor.named_parameters()}
    net.eval()
    x = image()
    with torch.no_grad():
        outs = net(x)
    arrays = {
        "shapes_json": np.array(json.dumps({k: list(v.shape) for k, v in extractor.state_dict().items()})),
        "init_sums_json": np.array(json.dumps(init_sums)),
        "grad_json": np.array(json.dumps(grads)),
        "num_channels_json": np.array(json.dumps(list(net.num_channels))),
        "image": x.numpy(),
    }
    for k, v in outs.items():
        arrays[f"out.{k}"] = v.contiguous().numpy()
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {len(extractor.state_dict())} keys, outputs {[tuple(v.shape) for v in outs.values()]} "
          f"(strides {[v.stride() for v in outs.values()]}), {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
