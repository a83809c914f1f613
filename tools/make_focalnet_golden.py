"""TEST INFRASTRUCTURE ONLY -- golden fixture of the FocalNet-L backbone, made by running the UNMODIFIED reference on the CPU.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_focalnet_golden.py

  focalnet_l_backbone.npz
    shapes_json        the reference backbone's state-dict keys and shapes (FocalNetBackbone("focalnet_large_lrf_fl4",
                       return_indices=(1, 2, 3), freeze_indices=(0,)): the feature extractor under "0.", the post-process norms
                       under "1.")
    init_sums_json     per-tensor sums of the reference FocalNet's default initialisation (focalnet_large_lrf_fl4 settings) under
                       torch.manual_seed(0)
    grad_json          requires_grad of every parameter after freeze_indices=(0,)
    num_channels_json  the backbone's num_channels
    image              (2, 3, 61, 99): image 0 full, image 1 a 53 x 85 image zero-padded into the batch
    out.layers.1/2/3.blocks  the backbone's outputs on it with the synthetic.focalnet_weights(WEIGHT_SEED) weights, in eval mode

The image gives a 16 x 25 map after the stem (61 x 99 padded to 64 x 100), then 8 x 13, 4 x 7 and 2 x 4: the stem's ceil rule
and odd downsample widths.  The weights are passed as a state dict of the bare FocalNet, so nothing is downloaded.  The weights
and the image are regenerated from their seeds by weights() / image(), which the tests share.  The reference's own
FocalNetBackbone.__new__, load_checkpoint and load_state_dict run; only the third-party modules it imports and that are not
installed here are stubbed (make_backbone_golden's stubs).
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

OUT = os.path.join(ROOT, "tests", "golden", "focalnet_l_backbone.npz")
WEIGHT_SEED, IMAGE_SEED = 91, 92
ARCH, RETURN_INDICES, FREEZE_INDICES = "focalnet_large_lrf_fl4", (1, 2, 3), (0,)
FOCALNET_L_FL4 = dict(embed_dim=192, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                      focal_levels=(4, 4, 4, 4), focal_windows=(3, 3, 3, 3), use_conv_embed=True, use_postln=True,
                      use_postln_in_modulation=False, use_layerscale=True, normalize_modulator=True)


def weights(state):
    """the fixture's weights for the network's state dict (synthetic.focalnet_weights)"""
    from salience_detr_b200 import synthetic

    return synthetic.focalnet_weights(state, WEIGHT_SEED)


def image():
    """(2, 3, 61, 99): a full image and a 53 x 85 one zero-padded to the batch size"""
    g = torch.Generator().manual_seed(IMAGE_SEED)
    x = torch.zeros(2, 3, 61, 99)
    x[0] = torch.randn(3, 61, 99, generator=g)
    x[1, :, :53, :85] = torch.randn(3, 53, 85, generator=g)
    return x


def main():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "backbones", "focalnet.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the original project")
    sys.path.insert(0, ref)
    _stub_missing_modules()
    from models.backbones.focalnet import FocalNet, FocalNetBackbone

    torch.manual_seed(0)
    init = FocalNet(**FOCALNET_L_FL4)
    state = init.state_dict()
    init_sums = {k: float(v.double().sum()) for k, v in state.items()}
    w = weights(state)
    del init

    net = FocalNetBackbone.__new__(FocalNetBackbone, ARCH, weights=w, return_indices=RETURN_INDICES,
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
        arrays[f"out.{k}"] = v.contiguous().numpy()
    np.savez_compressed(OUT, **arrays)
    print(f"wrote {OUT}: {len(net.state_dict())} keys, outputs {[tuple(v.shape) for v in outs.values()]}, "
          f"{os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
