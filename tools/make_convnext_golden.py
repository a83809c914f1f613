"""TEST INFRASTRUCTURE ONLY -- golden fixture of the ConvNeXt-L backbone, made by running the UNMODIFIED reference on the CPU.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_convnext_golden.py

  convnext_l_backbone.npz
    shapes_json        the reference feature extractor's state-dict keys and shapes (ConvNeXtBackbone("conv_l",
                       return_indices=(1, 2, 3), freeze_indices=(0,)))
    init_sums_json     per-tensor sums of the reference ConvNeXt's default initialisation (conv_l settings) under
                       torch.manual_seed(0), all keys but classifier.*
    grad_json          requires_grad of every parameter after freeze_indices=(0,)
    num_channels_json  the extractor's num_channels
    image              (2, 3, 64, 96): image 0 full, image 1 a 56 x 80 image zero-padded into the batch
    out.features.3/5/7 the extractor's outputs on it with the synthetic.convnext_weights(WEIGHT_SEED) weights, in eval mode

The weights are passed as a state dict, so nothing is downloaded.  The weights and the image are regenerated from their seeds by
weights() / image(), which the tests share.  The reference's own ConvNeXtBackbone.__new__, load_checkpoint and load_state_dict
run; only the third-party modules it imports and that are not installed here are stubbed (make_backbone_golden's stubs).
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

from tools.make_backbone_golden import _stub_missing_modules, image  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "convnext_l_backbone.npz")
WEIGHT_SEED = 71
RETURN_INDICES, FREEZE_INDICES = (1, 2, 3), (0,)


def weights(shapes):
    """the fixture's weights for a {key: shape} table (synthetic.convnext_weights)"""
    from salience_detr_b200 import synthetic

    return synthetic.convnext_weights(shapes, WEIGHT_SEED)


def main():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "backbones", "convnext.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the original project")
    sys.path.insert(0, ref)
    _stub_missing_modules()
    from models.backbones.convnext import CNBlockConfig, ConvNeXt, ConvNeXtBackbone

    setting = [CNBlockConfig(192, 384, 3), CNBlockConfig(384, 768, 3), CNBlockConfig(768, 1536, 27), CNBlockConfig(1536, None, 3)]
    torch.manual_seed(0)
    init = ConvNeXt(block_setting=setting, stochastic_depth_prob=0.5)
    init_sums = {k: float(v.double().sum()) for k, v in init.state_dict().items() if not k.startswith("classifier.")}
    shapes = {k: list(v.shape) for k, v in init.state_dict().items() if not k.startswith("classifier.")}
    del init

    net = ConvNeXtBackbone.__new__(ConvNeXtBackbone, "conv_l", weights=weights(shapes), return_indices=RETURN_INDICES,
                                   freeze_indices=FREEZE_INDICES)
    grads = {k: p.requires_grad for k, p in net.named_parameters()}
    net.eval()
    x = image()
    with torch.no_grad():
        outs = net(x)
    arrays = {
        "shapes_json": np.array(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()})),
        "init_sums_json": np.array(json.dumps(init_sums)),
        "grad_json": np.array(json.dumps(grads)),
        "num_channels_json": np.array(json.dumps(list(net.num_channels))),
        "image": x.numpy(),
    }
    for k, v in outs.items():
        arrays[f"out.{k}"] = v.numpy()
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {len(shapes)} keys, outputs {[tuple(v.shape) for v in outs.values()]}, "
          f"{os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
