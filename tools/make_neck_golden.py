"""TEST INFRASTRUCTURE ONLY -- golden fixtures of the RepVGG-PluX neck, made by running the UNMODIFIED reference.

    SDETR_REFERENCE_ROOT=<root of the original project> python tools/make_neck_golden.py

  neck_repnet.npz        RepVGGPluXNetwork([256]*4, [256]*4, BatchNorm2d, SiLU, groups=4) of models/necks/repnet.py on seeded
                         maps at the HALF geometry's level shapes (oracle/make_golden.py): eval outputs at sampled token rows,
                         one train-mode forward (sampled output rows and the updated running statistics of a few BatchNorm
                         layers), the key / shape list; and a RepVggPluXBlock with alpha=True (eval output, sampled).
  transformer_neck.npz   the HALF transformer (encoder, this neck, decoder) on the HALF inputs: the 5-tuple of
                         SalienceTransformer.forward and the decoder's `value` input at sampled token rows.

The weights are not stored: neck_state_dict() regenerates them from (sorted name, shape, seed), and the tests load the same
tensors.  The encoder / decoder weights are oracle.deterministic_state_dict(..., HALF_SEED), as for decoder_half_*.npz.
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
from oracle import make_golden as mg  # noqa: E402
from oracle import oracle as orc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
NECK_SEED, BLOCK_SEED, NECK_INPUT_SEED, NECK_ROWS = 41, 42, 43, 128
CHANNELS, GROUPS = 256, 4
# level shapes of the HALF inputs (480 x 640 images, strides 8, 16, 32, 64)
HALF_SHAPES = [(60, 80), (30, 40), (15, 20), (8, 10)]
TRAIN_STATS = ["lateral_convs.0.1", "layer_blocks.0.bottlenecks.1.conv1.1", "downsample_blocks.2.1", "pan_blocks.2.conv2.1"]


def neck_state_dict(shapes, seed):
    """Non-trivial neck weights from (sorted name order, shape, seed): convolution weights N(0, 1 / fan_in) with fan_in =
    prod(shape[1:]), BatchNorm gains 1 + 0.1 N, shifts and running means 0.1 N, running variances in [0.5, 1.5), biases 0.1 N,
    alpha 1 + 0.3 N, num_batches_tracked 7."""
    out = {}
    for i, name in enumerate(sorted(shapes)):
        g = torch.Generator().manual_seed(seed * 100003 + i)
        shp = tuple(int(v) for v in shapes[name])
        if name.endswith("num_batches_tracked"):
            out[name] = torch.tensor(7, dtype=torch.int64)
            continue
        x = torch.randn(shp, generator=g)
        if name.endswith("running_var"):
            x = 0.5 + torch.rand(shp, generator=g)
        elif name.endswith("alpha"):
            x = 1.0 + 0.3 * x
        elif len(shp) == 4:
            x = x / float(np.prod(shp[1:])) ** 0.5
        elif name.endswith(".weight"):
            x = 1.0 + 0.1 * x
        else:
            x = 0.1 * x
        out[name] = x
    return out


def neck_inputs(b=2, seed=NECK_INPUT_SEED):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(b, CHANNELS, h, w, generator=g) for h, w in HALF_SHAPES]


def block_input(seed=BLOCK_SEED):
    return torch.randn(2, CHANNELS, 13, 21, generator=torch.Generator().manual_seed(seed + 1))


def tokens(maps):
    return torch.cat([m.flatten(2).transpose(1, 2) for m in maps], 1)


def make_neck_repnet(ref):
    from collections import OrderedDict

    net = ref.repnet.RepVGGPluXNetwork([CHANNELS] * 4, [CHANNELS] * 4, groups=GROUPS, norm_layer=torch.nn.BatchNorm2d,
                                       activation=torch.nn.SiLU)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(neck_state_dict(shapes, NECK_SEED), strict=True)
    feats = neck_inputs()
    with torch.no_grad():
        ev = tokens(list(net.eval()(OrderedDict(enumerate(feats))).values()))
        tr = tokens(list(net.train()(OrderedDict(enumerate(feats))).values()))
    rows, ev_rows = mg.sample_rows(ev, NECK_ROWS, 700)
    res = dict(shapes_json=np.array(json.dumps({k: list(v) for k, v in shapes.items()})), rows_index=mg.np_(rows),
               eval_rows=mg.np_(ev_rows), eval_absmax=np.float32(ev.abs().max().item()),
               train_rows=mg.np_(torch.gather(tr, 1, rows[..., None].expand(-1, -1, CHANNELS))))
    sd = net.state_dict()
    for name in TRAIN_STATS:
        res[f"train.{name}.running_mean"] = mg.np_(sd[name + ".running_mean"])
        res[f"train.{name}.running_var"] = mg.np_(sd[name + ".running_var"])
        res[f"train.{name}.num_batches_tracked"] = mg.np_(sd[name + ".num_batches_tracked"])
    blk = ref.repnet.RepVggPluXBlock(CHANNELS, CHANNELS, activation_layer=torch.nn.SiLU, groups=GROUPS, alpha=True)
    bshapes = {k: tuple(v.shape) for k, v in blk.state_dict().items()}
    blk.load_state_dict(neck_state_dict(bshapes, BLOCK_SEED), strict=True)
    with torch.no_grad():
        bout = blk.eval()(block_input())
    res["block_shapes_json"] = np.array(json.dumps({k: list(v) for k, v in bshapes.items()}))
    res["block_out_idx"], res["block_out"], res["block_out_absmax"] = mg.sample_flat(bout, 4096, 701)
    np.savez_compressed(os.path.join(OUT, "neck_repnet.npz"), **res)


def make_transformer_neck(ref):
    tr, shapes = mg.half_reference()
    tr.neck = ref.repnet.RepVGGPluXNetwork([CHANNELS] * 4, [CHANNELS] * 4, groups=GROUPS, norm_layer=torch.nn.BatchNorm2d,
                                           activation=torch.nn.SiLU)
    nshapes = {k: tuple(v.shape) for k, v in tr.neck.state_dict().items()}
    tr.neck.load_state_dict(neck_state_dict(nshapes, NECK_SEED), strict=True)
    tr.eval()
    feats, masks, pos = orc.synthetic_inputs(mg.image_sizes(False), (480, 640), 256, seed=mg.HALF_INPUT_SEED)
    cap = {}
    dec_fwd = tr.decoder.forward

    def spy(**kw):
        cap["value"] = kw["value"]
        return dec_fwd(**kw)

    tr.decoder.forward = spy
    with torch.no_grad():
        full = tr(feats, masks, pos, None, None, None)
    del tr.decoder.forward
    rows, vals = mg.sample_rows(cap["value"], mg.HALF_ROWS, 300)
    res = dict(shapes_json=np.array(json.dumps({k: list(v) for k, v in shapes.items()})), value_rows_index=mg.np_(rows),
               value_rows=mg.np_(vals), value_absmax=np.float32(cap["value"].abs().max().item()))
    for i, t in enumerate(full[:4]):
        res[f"full{i}"] = mg.np_(t)
    for i, t in enumerate(full[4]):
        res[f"full_score{i}"] = mg.np_(t)
    np.savez_compressed(os.path.join(OUT, "transformer_neck.npz"), **res)


def main():
    from oracle import ref_import

    ref = ref_import.load()
    if ref.repnet is None:
        raise RuntimeError("the original project's models/necks/repnet.py could not be imported")
    make_neck_repnet(ref)
    make_transformer_neck(ref)
    for f in ("neck_repnet.npz", "transformer_neck.npz"):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    main()
