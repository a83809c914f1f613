"""TEST INFRASTRUCTURE ONLY -- golden fixture of the ResNet-50 backbone, made by running the UNMODIFIED reference on the CPU.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_backbone_golden.py

  resnet50_backbone.npz
    shapes_json      the reference feature extractor's state-dict keys and shapes (ResNetBackbone("resnet50",
                     norm_layer=FrozenBatchNorm2d, return_indices=(1, 2, 3), freeze_indices=(0,)))
    init_sums_json   per-tensor sums of the reference ResNet's default initialisation under torch.manual_seed(0)
                     (ResNet(block=Bottleneck, layers=(3, 4, 6, 3), norm_layer=FrozenBatchNorm2d), all keys but fc.*)
    grad_json        requires_grad of every parameter after freeze_indices=(0,)
    image            (2, 3, 64, 96): image 0 full, image 1 a 56 x 80 image zero-padded into the batch
    out.layer2/3/4   the extractor's outputs on it with the synthetic.resnet_weights(WEIGHT_SEED) weights

The weights and the image are regenerated from their seeds by weights() / image(), which the tests share.  The reference's own
ResNetBackbone.__new__, FrozenBatchNorm2d, load_checkpoint and load_state_dict run; only the third-party modules it imports
and that are not installed here (omegaconf, accelerate, terminaltables) are stubbed.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "resnet50_backbone.npz")
WEIGHT_SEED, IMAGE_SEED = 61, 62
RETURN_INDICES, FREEZE_INDICES = (1, 2, 3), (0,)


def weights(shapes):
    """the fixture's weights for a {key: shape} table (synthetic.resnet_weights)"""
    from salience_detr_b200 import synthetic

    return synthetic.resnet_weights(shapes, WEIGHT_SEED)


def image():
    """(2, 3, 64, 96): a full image and a 56 x 80 one zero-padded to the batch size (image_list_from_tensors' layout)"""
    g = torch.Generator().manual_seed(IMAGE_SEED)
    x = torch.zeros(2, 3, 64, 96)
    x[0] = torch.randn(3, 64, 96, generator=g)
    x[1, :, :56, :80] = torch.randn(3, 56, 80, generator=g)
    return x


def _stub_missing_modules():
    """omegaconf.DictConfig (a dict with attribute reads), OmegaConf.to_object (the identity), accelerate.logging.get_logger,
    terminaltables.AsciiTable"""
    import logging

    class DictConfig(dict):
        _metadata = types.SimpleNamespace(object_type=None)

        def __init__(self, content=None, flags=None):
            super().__init__(content or {})

        def __getattr__(self, name):
            try:
                return self[name]
            except KeyError as e:
                raise AttributeError(name) from e

    class OmegaConf:
        @staticmethod
        def to_object(cfg):
            return cfg  # the stub's configs are plain dicts and lists already

    omegaconf = types.ModuleType("omegaconf")
    omegaconf.DictConfig, omegaconf.ListConfig, omegaconf.OmegaConf = DictConfig, type("ListConfig", (list,), {}), OmegaConf
    accelerate = types.ModuleType("accelerate")
    acc_logging = types.ModuleType("accelerate.logging")
    acc_logging.get_logger = logging.getLogger
    accelerate.logging = acc_logging
    terminaltables = types.ModuleType("terminaltables")
    terminaltables.AsciiTable = lambda rows: types.SimpleNamespace(table=str(rows), inner_footing_row_border=False)
    for name, mod in (("omegaconf", omegaconf), ("accelerate", accelerate), ("accelerate.logging", acc_logging),
                      ("terminaltables", terminaltables)):
        sys.modules.setdefault(name, mod)


def main():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "backbones", "resnet.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the original project")
    sys.path.insert(0, ref)
    _stub_missing_modules()
    from models.backbones.resnet import Bottleneck, ResNet, ResNetBackbone
    from models.bricks.misc import FrozenBatchNorm2d

    torch.manual_seed(0)
    init = ResNet(block=Bottleneck, layers=(3, 4, 6, 3), norm_layer=FrozenBatchNorm2d)
    init_sums = {k: float(v.double().sum()) for k, v in init.state_dict().items() if not k.startswith("fc.")}
    shapes = {k: list(v.shape) for k, v in init.state_dict().items() if not k.startswith("fc.")}

    net = ResNetBackbone.__new__(ResNetBackbone, "resnet50", weights=weights(shapes), return_indices=RETURN_INDICES,
                                 freeze_indices=FREEZE_INDICES, norm_layer=FrozenBatchNorm2d)
    net.eval()
    x = image()
    with torch.no_grad():
        outs = net(x)
    arrays = {
        "shapes_json": np.array(json.dumps({k: list(v.shape) for k, v in net.state_dict().items()})),
        "init_sums_json": np.array(json.dumps(init_sums)),
        "grad_json": np.array(json.dumps({k: p.requires_grad for k, p in net.named_parameters()})),
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
