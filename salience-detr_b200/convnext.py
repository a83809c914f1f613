"""ConvNeXt backbone (models/backbones/convnext.py:ConvNeXtBackbone of the original project), used by the ConvNeXt configs
(configs/salience_detr/salience_detr_convnext_l_800_1333.py).

``ConvNeXtBackbone(arch, weights, return_indices, freeze_indices, **kwargs)`` is an ``nn.Module`` whose ``features`` follow
torchvision's public ConvNeXt structure up to the last returned stage (the stem ``features.0``, stage ``i`` at
``features.{2i+1}``, the downsample after it at ``features.{2i+2}``; no ``classifier``, no ``avgpool``), so its ``state_dict``
has exactly the reference feature extractor's keys and shapes.  The full network is built and initialised as the reference
does it (``trunc_normal_(std=0.02)``, zero biases, ``layer_scale`` 1e-6) in the same RNG order, so a seed gives the reference's
tensors.  ``forward(x)`` returns ``{"features.{2i+1}": map}`` for ``i`` in ``return_indices``, in that order.

``forward`` is the reference's op chain in torch, ``forward_torch(x)``, whenever ``tokens_supported(x)`` does not hold: with
autograd, on the CPU, in train mode with a nonzero stochastic-depth probability, for norms or blocks other than the defaults,
and for stage widths that are not multiples of 64 (conv_t, conv_s).  Otherwise it is ``forward_tokens(x)``, on token rows
``(b, h*w, C)``:

- the stem (``sdetr_convnext_stem``): conv 4x4 / 4 and its LayerNorm2d in fp32 FMAs, read straight from the NCHW batch;
- per CNBlock 5 launches: the depthwise 7x7 and its LayerNorm (``sdetr_dwconv7x7_layernorm_tokens``, into a buffer of its
  own), the activation scale, ``pw1``, the scale of its output, and ``pw2`` with exact GELU applied as it loads, the bias,
  ``layer_scale`` and the residual in the epilogue, written over the block input in place (``sdetr_gemm_f16x3_ex``, the
  persistent 3xFP16 projection GEMM: fp32-class accuracy whatever ``allow_tf32`` says);
- per downsample 3 launches: the LayerNorm2d written space-to-depth (``sdetr_layernorm_tokens_s2d``), its scale, and the
  2x2 / stride-2 convolution as one GEMM with K = 4 Cin against the weight permuted to (Cout, 2, 2, Cin).

Each returned map is a channels-last NCHW view of its own ``(b, h*w, C)`` token buffer, which ``ChannelMapper`` reads in place.
The derived weights (both Linears' fp16 pairs, the permuted downsample weight, the depthwise weight as (49, C)) are cached per
parameter version through ``derived.cached``.  No host synchronisation: the call can be captured in a CUDA graph.
"""
from __future__ import annotations

from functools import partial
from typing import Any, Callable, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn
from torch.nn import functional as F
from torchvision.ops.stochastic_depth import StochasticDepth

from . import cabi
from .token_backbone import FeatureBackbone, tokens_ready


class LayerNorm2d(nn.LayerNorm):
    """LayerNorm over the channels of an NCHW map"""

    def forward(self, x: Tensor) -> Tensor:
        x = x.permute(0, 2, 3, 1)
        x = F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps)
        return x.permute(0, 3, 1, 2)


class Permute(nn.Module):
    def __init__(self, dims: List[int]):
        super().__init__()
        self.dims = dims

    def forward(self, x: Tensor) -> Tensor:
        return torch.permute(x, self.dims)


class CNBlock(nn.Module):
    def __init__(self, dim: int, layer_scale: float, stochastic_depth_prob: float,
                 norm_layer: Optional[Callable[..., nn.Module]] = None):
        super().__init__()
        norm_layer = norm_layer or partial(nn.LayerNorm, eps=1e-6)
        self.block = nn.Sequential(
            nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim, bias=True),
            Permute([0, 2, 3, 1]),
            norm_layer(dim),
            nn.Linear(in_features=dim, out_features=4 * dim, bias=True),
            nn.GELU(),
            nn.Linear(in_features=4 * dim, out_features=dim, bias=True),
            Permute([0, 3, 1, 2]),
        )
        self.layer_scale = nn.Parameter(torch.ones(dim, 1, 1) * layer_scale)
        self.stochastic_depth = StochasticDepth(stochastic_depth_prob, "row")

    def forward(self, input: Tensor) -> Tensor:
        result = self.layer_scale * self.block(input)
        result = self.stochastic_depth(result)
        result += input
        return result


class CNBlockConfig:
    def __init__(self, input_channels: int, out_channels: Optional[int], num_layers: int):
        self.input_channels, self.out_channels, self.num_layers = input_channels, out_channels, num_layers

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}(input_channels={self.input_channels}, out_channels={self.out_channels}, "
                f"num_layers={self.num_layers})")


class ConvNeXt(nn.Module):
    """torchvision's ConvNeXt (the reference's copy of it)"""

    def __init__(self, block_setting: List[CNBlockConfig], stochastic_depth_prob: float = 0.0, layer_scale: float = 1e-6,
                 num_classes: int = 1000, block: Optional[Callable[..., nn.Module]] = None,
                 norm_layer: Optional[Callable[..., nn.Module]] = None, **kwargs: Any):
        super().__init__()
        if not block_setting:
            raise ValueError("The block_setting should not be empty")
        if not (isinstance(block_setting, Sequence) and all(isinstance(s, CNBlockConfig) for s in block_setting)):
            raise TypeError("The block_setting should be List[CNBlockConfig]")
        block = block or CNBlock
        norm_layer = norm_layer or partial(LayerNorm2d, eps=1e-6)
        c0 = block_setting[0].input_channels
        layers: List[nn.Module] = [nn.Sequential(nn.Conv2d(3, c0, kernel_size=4, stride=4, padding=0, bias=True), norm_layer(c0))]
        total = sum(cnf.num_layers for cnf in block_setting)
        stage_block_id = 0
        for cnf in block_setting:
            stage: List[nn.Module] = []
            for _ in range(cnf.num_layers):
                sd_prob = stochastic_depth_prob * stage_block_id / (total - 1.0)
                stage.append(block(cnf.input_channels, layer_scale, sd_prob))
                stage_block_id += 1
            layers.append(nn.Sequential(*stage))
            if cnf.out_channels is not None:
                layers.append(nn.Sequential(norm_layer(cnf.input_channels),
                                            nn.Conv2d(cnf.input_channels, cnf.out_channels, kernel_size=2, stride=2)))
        self.features = nn.Sequential(*layers)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        last = block_setting[-1]
        c_last = last.out_channels if last.out_channels is not None else last.input_channels
        self.classifier = nn.Sequential(norm_layer(c_last), nn.Flatten(1), nn.Linear(c_last, num_classes))
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)


class _KBlock:
    """one CNBlock in kernel form: the depthwise weight as (49, C), its LayerNorm, both Linears as fp16 pairs with device scales,
    and layer_scale as (C,)"""

    def __init__(self, blk: CNBlock):
        dw, ln, l1, l2 = blk.block[0], blk.block[2], blk.block[3], blk.block[5]
        c = dw.out_channels
        self.dw_w, self.dw_b = dw.weight.detach().reshape(c, 49).t().contiguous(), dw.bias.detach()
        self.ln_w, self.ln_b, self.eps = ln.weight.detach(), ln.bias.detach(), ln.eps
        self.w1, self.b1 = cabi.split_f16_pair_dev(l1.weight.detach()), l1.bias.detach()
        self.w2, self.b2 = cabi.split_f16_pair_dev(l2.weight.detach()), l2.bias.detach()
        self.gamma = blk.layer_scale.detach().reshape(c)


class _KDown:
    """one downsample in kernel form: its LayerNorm2d and the 2x2 / stride-2 weight as the (Cout, 2 * 2 * Cin) fp16 pair of
    its (Cout, 2, 2, Cin) permutation"""

    def __init__(self, ds: nn.Sequential):
        ln, conv = ds[0], ds[1]
        self.ln_w, self.ln_b, self.eps = ln.weight.detach(), ln.bias.detach(), ln.eps
        w = conv.weight.detach()
        self.w = cabi.split_f16_pair_dev(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous())
        self.b = conv.bias.detach()


class ConvNeXtBackbone(FeatureBackbone):
    # name -> ConvNeXt arguments (the reference's model_arch table, without the download URLs)
    model_arch = {
        "conv_t": dict(block_setting=[CNBlockConfig(96, 192, 3), CNBlockConfig(192, 384, 3), CNBlockConfig(384, 768, 9),
                                      CNBlockConfig(768, None, 3)], stochastic_depth_prob=0.1),
        "conv_s": dict(block_setting=[CNBlockConfig(96, 192, 3), CNBlockConfig(192, 384, 3), CNBlockConfig(384, 768, 27),
                                      CNBlockConfig(768, None, 3)], stochastic_depth_prob=0.4),
        "conv_b": dict(block_setting=[CNBlockConfig(128, 256, 3), CNBlockConfig(256, 512, 3), CNBlockConfig(512, 1024, 27),
                                      CNBlockConfig(1024, None, 3)], stochastic_depth_prob=0.5),
        "conv_l": dict(block_setting=[CNBlockConfig(192, 384, 3), CNBlockConfig(384, 768, 3), CNBlockConfig(768, 1536, 27),
                                      CNBlockConfig(1536, None, 3)], stochastic_depth_prob=0.5),
    }
    network, skip_prefixes, kblock, kdown = ConvNeXt, ("classifier.",), _KBlock, _KDown

    def _config(self, arch: str, kwargs: dict) -> dict:
        return {**self.model_arch[arch], **kwargs}

    @staticmethod
    def _stage_channels(cfg: dict, i: int) -> int:
        return cfg["block_setting"][i].input_channels

    # ---- token-layout inference --------------------------------------------------------------------------------------
    def tokens_supported(self, x) -> bool:
        """True when forward_tokens can run this call: a CUDA fp32 NCHW-contiguous (b, 3, H, W) input whose every map is at least
        1x1, parameters fp32 on its device, nothing that needs a gradient (autograd off, or neither the input nor a parameter
        requires one), no active stochastic depth (train mode with p > 0), and layers_supported()."""
        if not tokens_ready(self, x):
            return False
        hw = (x.shape[2] // 4, x.shape[3] // 4)
        for _ in range(self._num_stages() - 1):
            hw = self._down_hw(hw)
        if hw[0] < 1 or hw[1] < 1:
            return False
        for i in range(self._num_stages()):
            if any(blk.stochastic_depth.training and blk.stochastic_depth.p > 0 for blk in self.features[2 * i + 1]
                   if isinstance(blk, CNBlock)):
                return False
        return self.layers_supported()

    def layers_supported(self) -> bool:
        """The layer half of tokens_supported: the default stem, CNBlocks and downsamples (LayerNorm2d / nn.LayerNorm with
        affine weights, exact GELU) with stage widths that are multiples of 64 up to 1536."""
        def ln_ok(n, cls, c):
            return (type(n) is cls and n.normalized_shape == (c,) and n.weight is not None and n.bias is not None)

        def width_ok(c):
            return c % 64 == 0 and 0 < c <= 1536

        stem = self.features[0]
        if not (type(stem) is nn.Sequential and len(stem) == 2 and type(stem[0]) is nn.Conv2d):
            return False
        conv = stem[0]
        c = conv.out_channels
        if (conv.kernel_size, conv.stride, conv.padding, conv.dilation, conv.groups) != ((4, 4), (4, 4), (0, 0), (1, 1), 1):
            return False
        if conv.in_channels != 3 or conv.bias is None or not width_ok(c) or not ln_ok(stem[1], LayerNorm2d, c):
            return False
        for i in range(self._num_stages()):
            for blk in self.features[2 * i + 1]:
                if type(blk) is not CNBlock or len(blk.block) != 7:
                    return False
                dw, ln, l1, act, l2 = blk.block[0], blk.block[2], blk.block[3], blk.block[4], blk.block[5]
                if type(dw) is not nn.Conv2d or (dw.in_channels, dw.out_channels, dw.groups) != (c, c, c) or dw.bias is None:
                    return False
                if (dw.kernel_size, dw.stride, dw.padding, dw.dilation) != ((7, 7), (1, 1), (3, 3), (1, 1)):
                    return False
                if dw.padding_mode != "zeros" or not ln_ok(ln, nn.LayerNorm, c):
                    return False
                if type(act) is not nn.GELU or act.approximate != "none":
                    return False
                if not (type(l1) is nn.Linear and type(l2) is nn.Linear and l1.bias is not None and l2.bias is not None):
                    return False
                if (l1.in_features, l1.out_features, l2.in_features, l2.out_features) != (c, 4 * c, 4 * c, c):
                    return False
                if tuple(blk.layer_scale.shape) != (c, 1, 1):
                    return False
            if i + 1 < self._num_stages():
                ds = self.features[2 * i + 2]
                if not (type(ds) is nn.Sequential and len(ds) == 2 and ln_ok(ds[0], LayerNorm2d, c) and type(ds[1]) is nn.Conv2d):
                    return False
                conv = ds[1]
                if (conv.kernel_size, conv.stride, conv.padding, conv.dilation, conv.groups) != ((2, 2), (2, 2), (0, 0), (1, 1), 1):
                    return False
                if conv.in_channels != c or conv.bias is None or not width_ok(conv.out_channels):
                    return False
                c = conv.out_channels
        return True

    def launches_per_forward(self) -> int:
        """library launches of one forward_tokens: the stem, 5 per CNBlock (dwconv + LayerNorm, scale, pw1, scale, pw2) and 3
        per downsample between kept stages (space-to-depth LayerNorm, scale, GEMM)"""
        n = 1
        for i in range(self._num_stages()):
            n += 5 * len(self.features[2 * i + 1]) + (3 if i + 1 < self._num_stages() else 0)
        return n

    @staticmethod
    def _block_tokens(k: _KBlock, t: Tensor, hw: Tuple[int, int]) -> Tensor:
        u = cabi.dwconv7x7_layernorm_tokens(t, hw, k.dw_w, k.dw_b, k.ln_w, k.ln_b, k.eps)
        h = cabi.gemm_f16x3_ex(u, cabi.pow2_scale(u, 12), *k.w1, k.b1)
        # t = t + gamma * (GELU(h) W2^T + b2): the block writes over its input, which only it reads
        return cabi.gemm_f16x3_ex(h, cabi.pow2_scale(h, 12), *k.w2, k.b2, act=cabi.ACT_GELU, col_scale=k.gamma, z=t, out=t)

    @staticmethod
    def _down_tokens(ds: _KDown, t: Tensor, hw: Tuple[int, int]) -> Tensor:
        r = cabi.layernorm_tokens_s2d(t, hw, ds.ln_w, ds.ln_b, ds.eps)
        return cabi.gemm_f16x3_ex(r, cabi.pow2_scale(r, 12), *ds.w, ds.b)

    @staticmethod
    def _down_hw(hw: Tuple[int, int]) -> Tuple[int, int]:
        return hw[0] // 2, hw[1] // 2
