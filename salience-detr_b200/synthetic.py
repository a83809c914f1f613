"""Synthetic encoder inputs of the reference's shapes (SURVEY.md 8(d)): there is no dataset or checkpoint in
this environment, so benchmarks and smoke tests feed seeded random feature maps of the COCO geometry.

Restates, for input generation only: the padded batch mask (models/detectors/base_detector.py:169-175,
util/misc.py:92-95), its nearest-neighbour resize per level (models/detectors/salience_detr.py:175) and
``PositionEmbeddingSine(normalize=True, offset=-0.5)`` (models/bricks/position_encoding.py:48-65,
configs/salience_detr/salience_detr_resnet50_800_1333.py:32)."""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import List, Mapping, Sequence, Tuple

import torch
from torch.nn import functional as F

CONFIGS = {
    # name: (image sizes per batch element, padded (H, W), strides)
    "cpu_512": ([(512, 512)], (512, 512), (8, 16, 32, 64)),                       # BASELINE.json configs[0]
    "resnet50_800_1333_bs2": ([(800, 1333)] * 2, (800, 1344), (8, 16, 32, 64)),   # configs[1] (the metric's config)
    "resnet50_800_1333_bs2_ragged": ([(800, 1333), (640, 1000)], (800, 1344), (8, 16, 32, 64)),
    "resnet50_5scale_bs2": ([(800, 1333)] * 2, (800, 1344), (4, 8, 16, 32)),      # stress: Nv = 89 250
}


def resnet_weights(shapes: Mapping[str, Sequence[int]], seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a ResNet state dict of the given key -> shape table (in its order): convolutions N(0, 2 / fan_in)
    (He scale), FrozenBatchNorm buffers away from the identity -- weight 1 + U(-0.25, 0.25), bias and running_mean N(0, 0.1^2),
    running_var U(0.5, 2) -- so that folding them into the convolutions is exercised."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for k, shape in shapes.items():
        shape = tuple(int(v) for v in shape)
        if len(shape) == 4:
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
        elif k.endswith("running_var"):
            t = torch.rand(shape, generator=g) * 1.5 + 0.5
        elif k.endswith("running_mean") or k.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("weight"):
            t = 1.0 + (torch.rand(shape, generator=g) - 0.5) * 0.5
        else:
            raise ValueError(f"resnet_weights: no rule for {k} {shape}")
        out[k] = t
    return out


def convnext_weights(shapes: Mapping[str, Sequence[int]], seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a ConvNeXt state dict of the given key -> shape table (in its order): convolution and Linear weights
    N(0, 1 / fan_in), their biases N(0, 0.1^2), LayerNorm affines away from (1, 0) -- weight 1 + U(-0.25, 0.25), bias
    N(0, 0.1^2) -- and layer_scale U(0.05, 1) per channel.  At the 1e-6 layer_scale of the initialisation every block is the
    identity to fp32 rounding, which would hide any error in it."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for k, shape in shapes.items():
        shape = tuple(int(v) for v in shape)
        if k.endswith("layer_scale"):
            t = 0.05 + torch.rand(shape, generator=g) * 0.95
        elif len(shape) >= 2:
            t = torch.randn(shape, generator=g) / math.sqrt(math.prod(shape[1:]))
        elif k.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("weight"):
            t = 1.0 + (torch.rand(shape, generator=g) - 0.5) * 0.5
        else:
            raise ValueError(f"convnext_weights: no rule for {k} {shape}")
        out[k] = t
    return out


def swin_weights(state: Mapping[str, torch.Tensor], seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a V1 Swin Transformer state dict (in its order): Linear and convolution weights N(0, 1 / fan_in), their
    biases N(0, 0.1^2), LayerNorm affines away from (1, 0) -- weight 1 + U(-0.25, 0.25), bias N(0, 0.1^2) -- and every
    relative_position_bias_table N(0, 1), a spread that moves the softmax: at the 0.02 of the initialisation a wrong bias index
    would go unseen.  The relative_position_index buffers are copied from ``state``, the network's own state dict."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for k, v in state.items():
        shape = tuple(v.shape)
        if k.endswith("relative_position_index"):
            t = v.clone()
        elif k.endswith("relative_position_bias_table"):
            t = torch.randn(shape, generator=g)
        elif len(shape) >= 2:
            t = torch.randn(shape, generator=g) / math.sqrt(math.prod(shape[1:]))
        elif k.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("weight"):
            t = 1.0 + (torch.rand(shape, generator=g) - 0.5) * 0.5
        else:
            raise ValueError(f"swin_weights: no rule for {k} {shape}")
        out[k] = t
    return out


def focalnet_weights(state: Mapping[str, torch.Tensor], seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights for a FocalNet state dict (in its order), swin_weights' rules -- Linear and convolution weights
    N(0, 1 / fan_in), biases N(0, 0.1^2), LayerNorm weights 1 + U(-0.25, 0.25) -- with the layer scales gamma_1 / gamma_2
    U(0.05, 1): at their 1e-4 initialisation every block is nearly the identity, which would hide an error in it."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for k, v in state.items():
        shape = tuple(v.shape)
        if k.endswith(("gamma_1", "gamma_2")):
            t = 0.05 + torch.rand(shape, generator=g) * 0.95
        elif len(shape) >= 2:
            t = torch.randn(shape, generator=g) / math.sqrt(math.prod(shape[1:]))
        elif k.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.1
        elif k.endswith("weight"):
            t = 1.0 + (torch.rand(shape, generator=g) - 0.5) * 0.5
        else:
            raise ValueError(f"focalnet_weights: no rule for {k} {shape}")
        out[k] = t
    return out


def level_shapes(h: int, w: int, strides: Sequence[int]) -> List[Tuple[int, int]]:
    out: List[Tuple[int, int]] = []
    for i, s in enumerate(strides):
        if i == len(strides) - 1 and out and s == 2 * strides[i - 1]:
            ph, pw = out[-1]  # extra level = 3x3 stride-2 conv on the previous map (necks/channel_mapper.py:43-58)
            out.append(((ph - 1) // 2 + 1, (pw - 1) // 2 + 1))
        else:
            out.append((math.ceil(h / s), math.ceil(w / s)))
    return out


def sine_position_embedding(mask: torch.Tensor, num_pos_feats: int, temperature: float = 10000.0,
                            scale: float = 2 * math.pi, eps: float = 1e-6, offset: float = -0.5) -> torch.Tensor:
    keep = (~mask).to(torch.float32)
    y, x = keep.cumsum(1), keep.cumsum(2)
    y = (y + offset) / (y[:, -1:, :] + eps) * scale
    x = (x + offset) / (x[:, :, -1:] + eps) * scale
    dim_t = temperature ** (2 * torch.arange(num_pos_feats, device=mask.device).div(2, rounding_mode="floor")
                            / num_pos_feats)
    px, py = x[..., None] / dim_t, y[..., None] / dim_t
    px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=4).flatten(3)
    py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=4).flatten(3)
    return torch.cat((py, px), dim=3).permute(0, 3, 1, 2).contiguous()


def make_inputs(config: str = "resnet50_800_1333_bs2", embed_dim: int = 256, seed: int = 0, device="cpu"):
    """-> (feats, masks, pos): lists over levels of (b,C,H,W) f32, (b,H,W) bool, (b,C,H,W) f32."""
    sizes, (H, W), strides = CONFIGS[config]
    g = torch.Generator().manual_seed(seed)
    b = len(sizes)
    full = torch.ones(b, H, W, dtype=torch.bool)
    for i, (h, w) in enumerate(sizes):
        full[i, :h, :w] = False
    feats, masks, pos = [], [], []
    for (h, w) in level_shapes(H, W, strides):
        feats.append(torch.randn(b, embed_dim, h, w, generator=g).to(device))
        m = F.interpolate(full[None].float(), size=(h, w))[0].to(torch.bool).to(device)
        masks.append(m)
        pos.append(sine_position_embedding(m, embed_dim // 2))
    return feats, masks, pos


def build_model(embed_dim=256, d_ffn=2048, heads=8, levels=4, points=4, layers=6, num_classes=91,
                level_filter_ratio=(0.4, 0.8, 1.0, 1.0), layer_filter_ratio=(1.0, 0.8, 0.6, 0.6, 0.4, 0.2),
                topk_sa=300, max_num_embedding=None, strides=(8, 16, 32, 64), seed=0, learned_offsets=True):
    """Random-init encoder half with the geometry shared by all reference configs
    (configs/salience_detr/salience_detr_resnet50_800_1333.py:22-29,44-62,80-81).  ``learned_offsets`` perturbs
    the (zero-initialised) sampling-offset / attention-weight matrices so sampling is not just the init ring."""
    from .salience_transformer import SalienceTransformer, SalienceTransformerEncoder, SalienceTransformerEncoderLayer

    if max_num_embedding is None:  # 200 (salience_transformer.py:400); the 5-scale config raises it to 500 for its stride-4
        max_num_embedding = 500 if min(strides) < 8 else 200  # map (salience_detr_resnet50_5scale_800_1333.py:56)
    torch.manual_seed(seed)
    layer = SalienceTransformerEncoderLayer(embed_dim, d_ffn, 0.0, heads, torch.nn.ReLU(inplace=True), levels, points,
                                            topk_sa=topk_sa)
    enc = SalienceTransformerEncoder(layer, layers, max_num_embedding)
    tr = SalienceTransformer(enc, None, None, num_classes, levels, 900, tuple(level_filter_ratio),
                             tuple(layer_filter_ratio), level_strides=strides)
    if learned_offsets:
        with torch.no_grad():
            for l in enc.layers:
                l.self_attn.sampling_offsets.weight.normal_(0, 0.02)
                l.self_attn.attention_weights.weight.normal_(0, 0.5)
    return tr.eval()
