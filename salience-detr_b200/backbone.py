"""ResNet backbone (models/backbones/resnet.py:ResNetBackbone and models/bricks/misc.py:FrozenBatchNorm2d of the original
project), used by the ResNet configs (configs/salience_detr/salience_detr_resnet50_*.py).

``ResNetBackbone(arch, weights, return_indices, freeze_indices, **kwargs)`` is an ``nn.Module`` with the reference feature
extractor's sub-module names (``conv1``, ``bn1``, ``layer1`` ... up to the last returned stage, no ``fc``), so its
``state_dict`` has exactly the extractor's keys and shapes.  The network follows torchvision's public ResNet structure (ResNet
V1.5: the stride sits in a Bottleneck's 3x3 convolution) and its initialisation, in the same RNG order, so a seed gives the
reference's tensors.  ``forward(x)`` returns ``{"layer{i+1}": map}`` for ``i`` in ``return_indices``, in that order.

``forward`` is the reference's op chain in torch whenever ``tokens_supported(x)`` does not hold: with autograd, on the CPU, for
BasicBlock / ResNeXt / dilated / deformable networks and for norms other than this module's ``FrozenBatchNorm2d``.  Otherwise
it is ``forward_tokens(x)``: every FrozenBatchNorm folded into its convolution once per parameter / buffer version, the stem
(``sdetr_resnet_stem``, fp32 FMAs from the NCHW image batch), the max-pool (``sdetr_maxpool3x3s2_tokens``) and every
convolution on ``sdetr_conv2d_f16x3_ex`` (3xFP16 on wgmma, fp32-class accuracy whatever ``allow_tf32`` says) with ReLU and the
block's residual in the epilogue.  Each returned map is a channels-last NCHW view of its own ``(b, H*W, C)`` token buffer,
which ``ChannelMapper`` reads in place.  No host synchronisation: the call can be captured in a CUDA graph.
"""
from __future__ import annotations

from collections.abc import Mapping
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Type, Union

import torch
from torch import Tensor, nn

from . import cabi, derived
from .neck import _KConv


class FrozenBatchNorm2d(nn.Module):
    """BatchNorm2d with fixed statistics and affine parameters (all four are buffers): x * scale + (bias - running_mean *
    scale), scale = weight * rsqrt(running_var + eps).  ``num_batches_tracked`` in a loaded state dict is dropped."""

    def __init__(self, num_features: int, eps: float = 1e-5):
        super().__init__()
        self.eps = eps
        self.register_buffer("weight", torch.ones(num_features))
        self.register_buffer("bias", torch.zeros(num_features))
        self.register_buffer("running_mean", torch.zeros(num_features))
        self.register_buffer("running_var", torch.ones(num_features))

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        state_dict.pop(prefix + "num_batches_tracked", None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def forward(self, x: Tensor) -> Tensor:
        scale = self.weight.reshape(1, -1, 1, 1) * (self.running_var.reshape(1, -1, 1, 1) + self.eps).rsqrt()
        return x * scale + (self.bias.reshape(1, -1, 1, 1) - self.running_mean.reshape(1, -1, 1, 1) * scale)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}({self.weight.shape[0]}, eps={self.eps})"


class DeformConv2dPack(nn.Module):
    """A modulated deformable convolution used like a plain one: offsets and a sigmoid mask predicted from the input by two
    convolutions of the same geometry (zero-initialised), then torchvision's DeformConv2d."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int, stride: int = 1, padding: int = 0,
                 dilation: int = 1, groups: int = 1, bias: bool = True):
        super().__init__()
        from torchvision.ops import DeformConv2d

        k = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        self.in_channels, self.kernel_size, self.groups = in_channels, k, groups
        geo = dict(kernel_size=k, stride=stride, padding=padding, dilation=dilation, groups=groups, bias=True)
        self.conv_offset = nn.Conv2d(in_channels, groups * 2 * k[0] * k[1], **geo)
        self.conv_mask = nn.Conv2d(in_channels, groups * k[0] * k[1], **geo)
        self.deform_conv2d = DeformConv2d(in_channels, out_channels, k, stride=stride, padding=padding, dilation=dilation,
                                          groups=groups, bias=bias)
        for conv in (self.conv_offset, self.conv_mask):
            nn.init.zeros_(conv.weight)
            nn.init.zeros_(conv.bias)
        bound = 1.0 / (in_channels * k[0] * k[1]) ** 0.5
        nn.init.uniform_(self.deform_conv2d.weight, -bound, bound)
        if self.deform_conv2d.bias is not None:
            nn.init.zeros_(self.deform_conv2d.bias)

    def forward(self, x: Tensor) -> Tensor:
        return self.deform_conv2d(x, self.conv_offset(x), torch.sigmoid(self.conv_mask(x)))


def _conv3x3(cin: int, cout: int, stride: int = 1, groups: int = 1, dilation: int = 1, dcn: bool = False) -> nn.Module:
    return (DeformConv2dPack if dcn else nn.Conv2d)(cin, cout, kernel_size=3, stride=stride, padding=dilation, groups=groups,
                                                    bias=False, dilation=dilation)


def _conv1x1(cin: int, cout: int, stride: int = 1) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=1, stride=stride, bias=False)


class BasicBlock(nn.Module):
    expansion: int = 1

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None, groups: int = 1,
                 base_width: int = 64, dilation: int = 1, norm_layer: Optional[Callable[..., nn.Module]] = None,
                 with_dcn: bool = False):
        super().__init__()
        norm_layer = norm_layer or nn.BatchNorm2d
        if groups != 1 or base_width != 64:
            raise ValueError("BasicBlock only supports groups=1 and base_width=64")
        if dilation > 1:
            raise NotImplementedError("Dilation > 1 not supported in BasicBlock")
        self.conv1 = _conv3x3(inplanes, planes, stride)
        self.bn1 = norm_layer(planes)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = _conv3x3(planes, planes, dcn=with_dcn)
        self.bn2 = norm_layer(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x: Tensor) -> Tensor:
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        out += x if self.downsample is None else self.downsample(x)
        return self.relu(out)


class Bottleneck(nn.Module):
    expansion: int = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample: Optional[nn.Module] = None, groups: int = 1,
                 base_width: int = 64, dilation: int = 1, norm_layer: Optional[Callable[..., nn.Module]] = None,
                 with_dcn: bool = False):
        super().__init__()
        norm_layer = norm_layer or nn.BatchNorm2d
        width = int(planes * (base_width / 64.0)) * groups
        self.conv1 = _conv1x1(inplanes, width)
        self.bn1 = norm_layer(width)
        self.conv2 = _conv3x3(width, width, stride, groups, dilation, dcn=with_dcn)
        self.bn2 = norm_layer(width)
        self.conv3 = _conv1x1(width, planes * self.expansion)
        self.bn3 = norm_layer(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x: Tensor) -> Tensor:
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        out += x if self.downsample is None else self.downsample(x)
        return self.relu(out)


class ResNet(nn.Module):
    """torchvision's ResNet with the reference's extra ``stage_with_dcn`` argument (a deformable 3x3 per stage)."""

    def __init__(self, block: Type[Union[BasicBlock, Bottleneck]], layers: Sequence[int], num_classes: int = 1000,
                 zero_init_residual: bool = False, groups: int = 1, width_per_group: int = 64,
                 replace_stride_with_dilation: Optional[Sequence[bool]] = None, stage_with_dcn: Optional[Sequence[bool]] = None,
                 norm_layer: Optional[Callable[..., nn.Module]] = None):
        super().__init__()
        stage_with_dcn = stage_with_dcn or [False] * 4
        self._norm_layer = norm_layer = norm_layer or nn.BatchNorm2d
        self.inplanes, self.dilation = 64, 1
        replace_stride_with_dilation = replace_stride_with_dilation or [False, False, False]
        if len(replace_stride_with_dilation) != 3:
            raise ValueError("replace_stride_with_dilation should be None "
                             f"or a 3-element tuple, got {replace_stride_with_dilation}")
        self.groups, self.base_width = groups, width_per_group
        self.conv1 = nn.Conv2d(3, self.inplanes, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = norm_layer(self.inplanes)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, 64, layers[0], with_dcn=stage_with_dcn[0])
        for i, planes in enumerate((128, 256, 512)):
            setattr(self, f"layer{i + 2}", self._make_layer(block, planes, layers[i + 1], stride=2,
                                                            dilate=replace_stride_with_dilation[i], with_dcn=stage_with_dcn[i + 1]))
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck) and m.bn3.weight is not None:
                    nn.init.constant_(m.bn3.weight, 0)
                elif isinstance(m, BasicBlock) and m.bn2.weight is not None:
                    nn.init.constant_(m.bn2.weight, 0)

    def _make_layer(self, block, planes: int, blocks: int, stride: int = 1, dilate: bool = False, with_dcn: bool = False):
        norm_layer, downsample, previous_dilation = self._norm_layer, None, self.dilation
        if dilate:
            self.dilation *= stride
            stride = 1
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(_conv1x1(self.inplanes, planes * block.expansion, stride), norm_layer(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample, self.groups, self.base_width, previous_dilation, norm_layer,
                        with_dcn)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, groups=self.groups, base_width=self.base_width, dilation=self.dilation,
                                norm_layer=norm_layer, with_dcn=with_dcn))
        return nn.Sequential(*layers)


def _fold(conv: nn.Conv2d, bn: FrozenBatchNorm2d) -> Tuple[Tensor, Tensor]:
    """(W * scale, bias - running_mean * scale) in float64, scale = weight * rsqrt(running_var + eps)"""
    scale = bn.weight.double() * (bn.running_var.double() + bn.eps).rsqrt()
    return conv.weight.double() * scale.view(-1, 1, 1, 1), bn.bias.double() - bn.running_mean.double() * scale


class ResNetBackbone(nn.Module):
    # name -> ResNet arguments (the reference's model_arch table, without the download URLs)
    model_arch = {
        "resnet18": dict(block=BasicBlock, layers=(2, 2, 2, 2)),
        "resnet34": dict(block=BasicBlock, layers=(3, 4, 6, 3)),
        "resnet50": dict(block=Bottleneck, layers=(3, 4, 6, 3)),
        "resnet101": dict(block=Bottleneck, layers=(3, 4, 23, 3)),
        "resnet152": dict(block=Bottleneck, layers=(3, 8, 36, 3)),
        "resnext50_32x4d": dict(block=Bottleneck, layers=(3, 4, 6, 3), groups=32, width_per_group=4),
        "resnext101_32x4d": dict(block=Bottleneck, layers=(3, 4, 23, 3), groups=32, width_per_group=4),
        "resnext101_32x8d": dict(block=Bottleneck, layers=(3, 4, 23, 3), groups=32, width_per_group=8),
        "resnext101_64x4d": dict(block=Bottleneck, layers=(3, 4, 23, 3), groups=64, width_per_group=4),
        "wide_resnet50_2": dict(block=Bottleneck, layers=(3, 4, 6, 3), width_per_group=128),
        "wide_resnet101_2": dict(block=Bottleneck, layers=(3, 4, 23, 3), width_per_group=128),
    }

    def __init__(self, arch: str, weights=None, return_indices: Tuple[int, ...] = (0, 1, 2, 3), freeze_indices: Tuple = (),
                 **kwargs):
        super().__init__()
        if arch not in self.model_arch:
            raise ValueError(f"Expected architecture in {list(self.model_arch)} but got {arch}")
        cfg = {**self.model_arch[arch], **kwargs}
        resnet = ResNet(**cfg)
        self._load_weights(resnet, weights)
        if len(freeze_indices) > 0:
            for m in [resnet.conv1, resnet.bn1] + [resnet.get_submodule(f"layer{i + 1}") for i in freeze_indices]:
                m.eval()
                for p in m.parameters():
                    p.requires_grad = False
        self.return_indices = tuple(int(i) for i in return_indices)
        # the modules the feature extractor keeps: the stem and the stages up to the last returned one
        for name in ["conv1", "bn1", "relu", "maxpool"] + [f"layer{i + 1}" for i in range(max(self.return_indices) + 1)]:
            setattr(self, name, getattr(resnet, name))
        self.num_channels = [64 * cfg["block"].expansion * 2 ** i for i in self.return_indices]

    @staticmethod
    def _load_weights(resnet: ResNet, weights):
        """None: keep the initialisation.  A state dict (or one under "model"), or a local path read with torch.load: every key
        but fc.* must match the network exactly."""
        if weights is None:
            return
        if isinstance(weights, str):
            if weights.startswith(("http://", "https://")):
                raise RuntimeError(f"ResNetBackbone: downloading weights is not supported ({weights}); pass a state dict or "
                                   "a local file")
            weights = torch.load(weights, map_location="cpu")
        if not isinstance(weights, Mapping):
            raise TypeError(f"ResNetBackbone: weights must be None, a state dict or a path, got {type(weights).__name__}")
        if "model" in weights:
            weights = weights["model"]
        res = resnet.load_state_dict({k: v for k, v in weights.items() if not k.startswith("fc.")}, strict=False)
        missing = [k for k in res.missing_keys if not k.startswith("fc.")]
        if missing or res.unexpected_keys:
            raise RuntimeError(f"ResNetBackbone: weights do not match the network: missing {missing}, "
                               f"unexpected {res.unexpected_keys}")

    def _stages(self) -> List[nn.Sequential]:
        return [getattr(self, f"layer{i + 1}") for i in range(max(self.return_indices) + 1)]

    def forward(self, x: Tensor) -> Dict[str, Tensor]:
        if self.tokens_supported(x):
            return self.forward_tokens(x)
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        feats = []
        for layer in self._stages():
            x = layer(x)
            feats.append(x)
        return {f"layer{i + 1}": feats[i] for i in self.return_indices}

    # ---- token-layout inference --------------------------------------------------------------------------------------
    def tokens_supported(self, x) -> bool:
        """True when forward_tokens can run this call: a CUDA fp32 NCHW-contiguous (b, 3, H, W) input, parameters and buffers
        fp32 on its device, nothing that needs a gradient (autograd off, or neither the input nor a parameter requires one),
        and layers_supported()."""
        if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3):
            return False
        if x.numel() == 0 or not x.is_contiguous():
            return False
        if any(t.device != x.device or t.dtype != torch.float32 for t in list(self.parameters()) + list(self.buffers())):
            return False
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            return False
        return self.layers_supported()

    def layers_supported(self) -> bool:
        """The layer half of tokens_supported: Bottleneck blocks of plain convolutions with groups 1, dilation 1 and widths that
        are multiples of 64, and every norm exactly this module's FrozenBatchNorm2d."""
        if type(self.bn1) is not FrozenBatchNorm2d:
            return False
        for layer in self._stages():
            for blk in layer:
                if type(blk) is not Bottleneck:
                    return False
                convs = [blk.conv1, blk.conv2, blk.conv3] + ([blk.downsample[0]] if blk.downsample is not None else [])
                norms = [blk.bn1, blk.bn2, blk.bn3] + ([blk.downsample[1]] if blk.downsample is not None else [])
                if blk.downsample is not None and len(blk.downsample) != 2:
                    return False
                for conv in convs:
                    if type(conv) is not nn.Conv2d or conv.groups != 1 or conv.dilation != (1, 1) or conv.bias is not None:
                        return False
                    if conv.in_channels % 64 or conv.out_channels % 64:
                        return False
                if any(type(n) is not FrozenBatchNorm2d for n in norms):
                    return False
        return True

    def _kernel_weights(self):
        """the folded stem ((147, 64) weight, bias) and per stage per block the (conv1, conv2, conv3, downsample or None)
        convolutions in kernel form, rebuilt when any parameter or buffer changes"""
        def build():
            w, b = _fold(self.conv1, self.bn1)
            stem = (w.reshape(64, 147).t().float().contiguous(), b.float().contiguous())
            relu = cabi.ACT_RELU
            stages = []
            for layer in self._stages():
                blocks = []
                for blk in layer:
                    ds = blk.downsample
                    blocks.append((_KConv(*_fold(blk.conv1, blk.bn1), 1, 1, relu),
                                   _KConv(*_fold(blk.conv2, blk.bn2), 1, blk.conv2.stride[0], relu),
                                   _KConv(*_fold(blk.conv3, blk.bn3), 1, 1, relu),
                                   _KConv(*_fold(ds[0], ds[1]), 1, ds[0].stride[0], 0) if ds is not None else None))
                stages.append(blocks)
            return stem, stages
        return derived.cached(self, "kernel_weights", list(self.parameters()) + list(self.buffers()), build)

    def launches_per_forward(self) -> int:
        """library launches of one forward_tokens: the stem, the max-pool, and per convolution 2 (activation scale +
        convolution), where a block's conv1 and downsample share the scale of the tensor they both read"""
        n = 2
        for layer in self._stages():
            for blk in layer:
                n += 6 + (1 if blk.downsample is not None else 0)
        return n

    @staticmethod
    def _conv(k: _KConv, x: Tensor, hw, scale: Tensor, out=None, z=None) -> Tensor:
        return cabi.conv2d_f16x3(x, hw, scale, k.w_hi, k.w_lo, k.w_scale, k.bias, 1, k.ksize, k.stride, k.act, out=out, z=z)

    def forward_tokens(self, x: Tensor) -> Dict[str, Tensor]:
        """The backbone on ``x`` (b, 3, H, W) -> {"layer{i+1}": (b, C, h, w)} for i in return_indices, each a channels-last view
        (strides (h*w*C, 1, w*C, C)) of its own (b, h*w, C) token buffer; the values of forward() in torch.  No host
        synchronisation."""
        if not self.tokens_supported(x):
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported)")
        (stem_w, stem_b), stages = self._kernel_weights()
        b, _, H, W = x.shape
        hw = ((H - 1) // 2 + 1, (W - 1) // 2 + 1)
        t = cabi.resnet_stem(x, stem_w, stem_b)
        t = cabi.maxpool3x3s2_tokens(t, hw)
        hw = ((hw[0] - 1) // 2 + 1, (hw[1] - 1) // 2 + 1)
        feats = []
        for blocks in stages:
            for c1, c2, c3, ds in blocks:
                s = cabi.pow2_scale(t, 12)
                y1 = self._conv(c1, t, hw, s)
                y2 = self._conv(c2, y1, hw, cabi.pow2_scale(y1, 12))
                s2 = cabi.pow2_scale(y2, 12)
                hw2 = ((hw[0] - 1) // c2.stride + 1, (hw[1] - 1) // c2.stride + 1)
                # the residual is the downsample's fresh output, or a block input that only this block reads (an earlier block
                # of the same stage): conv3 writes over it in place
                ident = self._conv(ds, t, hw, s) if ds is not None else t
                t, hw = self._conv(c3, y2, hw2, s2, out=ident, z=ident), hw2
            feats.append((t, hw))
        outs = {}
        for i in self.return_indices:
            t, (h, w) = feats[i]
            outs[f"layer{i + 1}"] = t.unflatten(1, (h, w)).permute(0, 3, 1, 2)
        return outs
