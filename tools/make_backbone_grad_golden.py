"""TEST INFRASTRUCTURE ONLY -- golden fixture of the ResNet-50 backbone's training gradients, made by running the UNMODIFIED
reference on the CPU with the recipe of tools/make_backbone_golden.py.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_backbone_grad_golden.py

  resnet50_backbone_grads.npz
    names_json       the trainable parameters of ResNetBackbone("resnet50", norm_layer=FrozenBatchNorm2d,
                     return_indices=(1, 2, 3), freeze_indices=(0,)), in named_parameters() order
    sumsq            per parameter, the float64 sum of squares of its gradient
    dot              per parameter, the float64 dot product of its gradient with probe(name) (a seeded Gaussian)

The network and the image run in float64: the make_backbone_golden weights, its padded (2, 3, 64, 96) image, and the loss
sum_k sum(out_k * R_k) with R_k = cotangents() (seeded).  Two numbers per parameter keep the fixture small.
"""
from __future__ import annotations

import json
import os
import sys
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools import make_backbone_golden as mbg  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "resnet50_backbone_grads.npz")
COTANGENT_SEED = 63


def cotangents(outs):
    """R_k for each output map (same shape, float64, seeded in output order)"""
    g = torch.Generator().manual_seed(COTANGENT_SEED)
    return {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in outs.items()}


def probe(name, shape):
    """the seeded Gaussian the fixture dots a parameter's gradient with"""
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()))
    return torch.randn(shape, generator=g, dtype=torch.float64)


def gradient_stats(net, x):
    """{name: (sumsq, dot)} of every trainable parameter's gradient of sum_k sum(out_k * R_k), net and x in float64"""
    outs = net(x)
    loss = sum((v * r).sum() for v, r in zip(outs.values(), cotangents(outs).values()))
    names = [n for n, p in net.named_parameters() if p.requires_grad]
    grads = torch.autograd.grad(loss, [p for n, p in net.named_parameters() if p.requires_grad])
    return {n: (float((g * g).sum()), float((g * probe(n, g.shape)).sum())) for n, g in zip(names, grads)}


def main():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "backbones", "resnet.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the original project")
    sys.path.insert(0, ref)
    mbg._stub_missing_modules()
    from models.backbones.resnet import Bottleneck, ResNet, ResNetBackbone
    from models.bricks.misc import FrozenBatchNorm2d

    init = ResNet(block=Bottleneck, layers=(3, 4, 6, 3), norm_layer=FrozenBatchNorm2d)
    shapes = {k: list(v.shape) for k, v in init.state_dict().items() if not k.startswith("fc.")}
    net = ResNetBackbone.__new__(ResNetBackbone, "resnet50", weights=mbg.weights(shapes), return_indices=mbg.RETURN_INDICES,
                                 freeze_indices=mbg.FREEZE_INDICES, norm_layer=FrozenBatchNorm2d).double()
    stats = gradient_stats(net, mbg.image().double())
    names = list(stats)
    np.savez_compressed(OUT, names_json=np.array(json.dumps(names)), sumsq=np.array([stats[n][0] for n in names]),
                        dot=np.array([stats[n][1] for n in names]))
    print(f"wrote {OUT}: {len(names)} parameters, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
