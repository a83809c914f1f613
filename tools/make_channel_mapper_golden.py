"""TEST INFRASTRUCTURE ONLY -- golden fixture of the ChannelMapper input neck, made by running the UNMODIFIED reference.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_channel_mapper_golden.py

  channel_mapper.npz   ChannelMapper(in_channels=(128, 256, 512), out_channels=256, num_outs=4) of
                       models/necks/channel_mapper.py (GroupNorm(32), no activation: the reference default), built under
                       torch.manual_seed(MAPPER_SEED) -- so its xavier initialisation is the reference's own -- with the GroupNorm
                       gains / shifts then perturbed from AFFINE_SEED; its four outputs (bs=2, maps 12x20, 6x10, 3x5 and the extra
                       2x3 level) in full, and the key / shape list.

Inputs and weights are not stored: build() and inputs() regenerate them from the seeds, and the tests use the same functions.
"""
from __future__ import annotations

import json
import os
import sys
from collections import OrderedDict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "channel_mapper.npz")
MAPPER_SEED, AFFINE_SEED, INPUT_SEED = 51, 52, 53
IN_CHANNELS, OUT_CHANNELS, NUM_OUTS, BATCH = (128, 256, 512), 256, 4, 2
# odd map sizes: tile edges, a 3-row level, an extra level of 2x3, and H*W*4 not a multiple of 16 everywhere
SHAPES = [(12, 20), (6, 10), (3, 5)]


def perturb_affine(mapper):
    """GroupNorm gains 1 + 0.2 N and shifts 0.2 N from AFFINE_SEED (in module order), so the affine part is exercised."""
    g = torch.Generator().manual_seed(AFFINE_SEED)
    with torch.no_grad():
        for m in mapper.modules():
            if isinstance(m, torch.nn.GroupNorm):
                m.weight.copy_(1.0 + 0.2 * torch.randn(m.weight.shape, generator=g))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=g))
    return mapper


def build(cls):
    """``cls(IN_CHANNELS, OUT_CHANNELS, NUM_OUTS)`` constructed under torch.manual_seed(MAPPER_SEED), affine perturbed."""
    state = torch.random.get_rng_state()
    torch.manual_seed(MAPPER_SEED)
    try:
        mapper = cls(list(IN_CHANNELS), OUT_CHANNELS, NUM_OUTS)
    finally:
        torch.random.set_rng_state(state)
    return perturb_affine(mapper).eval()


def inputs(scale=1.0, b=BATCH):
    g = torch.Generator().manual_seed(INPUT_SEED)
    return OrderedDict((str(i), torch.randn(b, c, h, w, generator=g) * scale) for i, (c, (h, w)) in enumerate(zip(IN_CHANNELS, SHAPES)))


def main():
    from oracle import ref_import

    ref_import.load()  # puts the original project on sys.path
    from models.necks.channel_mapper import ChannelMapper

    mapper = build(ChannelMapper)
    with torch.no_grad():
        outs = mapper(inputs())
    res = dict(shapes_json=np.array(json.dumps({k: list(v.shape) for k, v in mapper.state_dict().items()})))
    for i, o in enumerate(outs):
        res[f"out{i}"] = o.detach().numpy().astype(np.float32)
    np.savez_compressed(OUT, **res)
    print(os.path.basename(OUT), os.path.getsize(OUT) // 1024, "KiB", [tuple(o.shape) for o in outs])


if __name__ == "__main__":
    main()
