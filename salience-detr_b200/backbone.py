"""ResNet backbone (models/backbones/resnet.py:ResNetBackbone and models/bricks/misc.py:FrozenBatchNorm2d of the original
project), used by the ResNet configs (configs/salience_detr/salience_detr_resnet50_*.py).

``ResNetBackbone(arch, weights, return_indices, freeze_indices, **kwargs)`` is an ``nn.Module`` with the reference feature
extractor's sub-module names (``conv1``, ``bn1``, ``layer1`` ... up to the last returned stage, no ``fc``), so its
``state_dict`` has exactly the extractor's keys and shapes.  The network follows torchvision's public ResNet structure (ResNet
V1.5: the stride sits in a Bottleneck's 3x3 convolution) and its initialisation, in the same RNG order, so a seed gives the
reference's tensors.  ``forward(x)`` returns ``{"layer{i+1}": map}`` for ``i`` in ``return_indices``, in that order.

``forward`` is the reference's op chain in torch whenever ``tokens_supported(x)`` does not hold: with autograd, on the CPU, for
BasicBlock / ResNeXt / dilated / deformable networks and for norms other than this module's ``FrozenBatchNorm2d``.  Otherwise
it is ``forward_tokens(x)``: every FrozenBatchNorm folded into its convolution on the device (``sdetr_frozen_bn_fold``, in
float64 with each operation rounded alone) once per parameter / buffer version, the stem (``sdetr_resnet_stem``, fp32 FMAs
from the NCHW image batch), the max-pool (``sdetr_maxpool3x3s2_tokens``) and every convolution a ``neck.TokenConv`` on
``sdetr_conv2d_f16x3`` (3xFP16 on wgmma, fp32-class accuracy whatever ``allow_tf32`` says) with ReLU and the block's residual
in the epilogue.  Each returned map is a channels-last NCHW view of its own ``(b, H*W, C)`` token buffer,
which ``ChannelMapper`` reads in place.  No host synchronisation: the call can be captured in a CUDA graph.

Under autograd, ``forward_tokens`` trains the convolutions of layers 1-4 in token layout when ``training_tokens_supported(x)``
holds (a frozen stem, an image that needs no gradient): one ``torch.autograd.Function`` over the blocks from the first one
with a trainable weight on.  Every call folds each FrozenBatchNorm into its convolution as inference does and splits it into
both fp16 layouts (``sdetr_conv2d_f16x3_split_weight``), so the forward writes the bits of the inference path and an
optimizer step between CUDA-graph replays is seen.  The backward runs the whole chain: input gradients on
``sdetr_conv2d_f16x3_dgrad`` with the residual sum (``z``) and the ReLU mask (``m``) in its epilogue, weight gradients on
``sdetr_conv2d_f16x3_wgrad`` with the FrozenBatchNorm scale in its write, and only the gradients something upstream needs.
``forward`` itself stays the torch chain under autograd.
"""
from __future__ import annotations

from collections.abc import Mapping
from typing import Callable, Dict, List, Optional, Sequence, Tuple, Type, Union

import torch
from torch import Tensor, nn

from . import cabi, derived
from .neck import TokenConv


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

    # ---- token-layout training -----------------------------------------------------------------------------------------
    def training_tokens_supported(self, x) -> bool:
        """True when forward_tokens can train this call in token layout: layers_supported() on a CUDA fp32 NCHW-contiguous
        (b, 3, H, W) input with parameters and buffers fp32 on its device, a frozen stem (conv1.weight needs no gradient), an
        input that needs no gradient, and autograd recording (grad enabled and some parameter requiring a gradient).  A stem
        weight gradient and image gradients need forward()."""
        if not _cuda_image(x) or x.requires_grad:
            return False
        if any(t.device != x.device or t.dtype != torch.float32 for t in list(self.parameters()) + list(self.buffers())):
            return False
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())) or self.conv1.weight.requires_grad:
            return False
        return self.layers_supported()

    def _train_plan(self):
        """(blocks, first, stage_end): the Bottlenecks of the kept stages in order, the index of the first one with a trainable
        convolution (the blocks before it neither train nor carry a gradient), and the index of each stage's last block"""
        blocks = [blk for layer in self._stages() for blk in layer]
        first = next(i for i, blk in enumerate(blocks) if any(c.weight.requires_grad for c in _block_convs(blk)))
        return blocks, first, self._stage_ends()

    def _stage_ends(self) -> List[int]:
        """the index of each kept stage's last Bottleneck, counting the blocks of all kept stages in order"""
        ends, n = [], 0
        for layer in self._stages():
            n += len(layer)
            ends.append(n - 1)
        return ends

    def _folded(self, dgrad_from: Optional[int] = None):
        """(stem, convs): every FrozenBatchNorm folded into its convolution on the device (sdetr_frozen_bn_fold).  stem: the
        folded (147, 64) weight and bias of sdetr_resnet_stem; convs: per Bottleneck of the kept stages in order, its (conv1,
        conv2, conv3, downsample or None) as TokenConvs with the FrozenBatchNorm scale for the weight gradient, the blocks from
        index ``dgrad_from`` on with the input-gradient weights too"""
        w, _, b = cabi.frozen_bn_fold(self.conv1.weight.detach().contiguous(), self.bn1, scale=False)
        stem = (w.view(64, 147).t().contiguous(), b)

        def conv(c: nn.Conv2d, bn: FrozenBatchNorm2d, act: int, dgrad: bool) -> TokenConv:
            wf, scale, bias = cabi.frozen_bn_fold(c.weight.detach().contiguous(), bn)
            return TokenConv(wf, bias, 1, c.stride[0], act, dgrad, scale)

        relu, convs = cabi.ACT_RELU, []
        for j, blk in enumerate(blk for layer in self._stages() for blk in layer):
            d, ds = dgrad_from is not None and j >= dgrad_from, blk.downsample
            convs.append((conv(blk.conv1, blk.bn1, relu, d), conv(blk.conv2, blk.bn2, relu, d), conv(blk.conv3, blk.bn3, relu, d),
                          conv(ds[0], ds[1], 0, d) if ds is not None else None))
        return stem, convs

    def launches_per_training_step(self) -> int:
        """library launches of one forward_tokens under autograd and its backward (training_tokens_supported): the stem's fold,
        the stem and the max-pool; per convolution 3 (fold, weight scale, split); per block the forward's 6 (+1 downsample);
        per block from the first trainable one, backwards: the scale of G, and per gradient it needs 1 per input gradient, 1 per
        activation scale of an input gradient a weight gradient reads, and 2 per weight gradient (convolution + split sum)"""
        blocks, first, _ = self._train_plan()
        n = 3
        for blk in blocks:
            ds = blk.downsample is not None
            n += 3 * (3 + ds) + 6 + ds
        for j in range(first, len(blocks)):
            blk, need_in = blocks[j], j > first
            c1, c2, c3 = (c.weight.requires_grad for c in (blk.conv1, blk.conv2, blk.conv3))
            ds = blk.downsample is not None
            n += 1 + 2 * c3 + (2 * blk.downsample[0].weight.requires_grad if ds else 0)
            if c2 or c1 or need_in:
                n += 2 + 2 * c2
                if c1 or need_in:
                    n += 2 + 2 * c1
            if need_in:
                n += 1 + ds
        return n

    def _train_tokens(self, x: Tensor) -> Dict[str, Tensor]:
        """forward_tokens under autograd (training_tokens_supported): the blocks before the first trainable one as in inference,
        the rest through _TrainBlocks; the same channels-last views, with the bits of the inference path"""
        blocks, first, stage_end = self._train_plan()
        stem, ks = self._folded(dgrad_from=first)
        t, hw = _stem(x, stem)
        feats = {}
        for j in range(first):  # as in inference: nothing saved
            t, hw = _bottleneck(ks[j], t, hw)
            if j in stage_end:
                feats[stage_end.index(j)] = (t, hw)
        trainable = [[c.weight.requires_grad for c in _block_convs(blk)] for blk in blocks[first:]]
        weights = [c.weight for blk in blocks[first:] for c in _block_convs(blk) if c.weight.requires_grad]
        ends = [stage_end.index(j) if j in stage_end and stage_end.index(j) in self.return_indices else None
                for j in range(first, len(blocks))]
        run = _TrainRun(ks[first:], trainable, ends, hw)
        outs = _TrainBlocks.apply(run, t, *weights)
        for i, o in zip(run.returned, outs):
            feats[i] = (o, run.out_hw[i])
        res = {}
        for i in self.return_indices:
            t, (h, w) = feats[i]
            res[f"layer{i + 1}"] = t.unflatten(1, (h, w)).permute(0, 3, 1, 2)
        return res

    def _kernel_weights(self):
        """_folded() for inference, rebuilt when any parameter or buffer changes"""
        return derived.cached(self, "kernel_weights", list(self.parameters()) + list(self.buffers()), self._folded)

    def launches_per_forward(self) -> int:
        """library launches of one forward_tokens: the stem, the max-pool, and per convolution 2 (activation scale +
        convolution), where a block's conv1 and downsample share the scale of the tensor they both read"""
        n = 2
        for layer in self._stages():
            for blk in layer:
                n += 6 + (1 if blk.downsample is not None else 0)
        return n

    def forward_tokens(self, x: Tensor) -> Dict[str, Tensor]:
        """The backbone on ``x`` (b, 3, H, W) -> {"layer{i+1}": (b, C, h, w)} for i in return_indices, each a channels-last view
        (strides (h*w*C, 1, w*C, C)) of its own (b, h*w, C) token buffer; the values of forward() in torch.  No host
        synchronisation."""
        if not self.tokens_supported(x):
            if self.training_tokens_supported(x):
                return self._train_tokens(x)
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported)")
        stem, convs = self._kernel_weights()
        t, hw = _stem(x, stem)
        feats, stage_end = [], self._stage_ends()
        for j, ks in enumerate(convs):
            t, hw = _bottleneck(ks, t, hw)
            if j in stage_end:
                feats.append((t, hw))
        outs = {}
        for i in self.return_indices:
            t, (h, w) = feats[i]
            outs[f"layer{i + 1}"] = t.unflatten(1, (h, w)).permute(0, 3, 1, 2)
        return outs


def _cuda_image(x) -> bool:
    """a non-empty NCHW-contiguous CUDA fp32 (b, 3, H, W) tensor"""
    return (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.numel() > 0
            and x.is_contiguous())


def _block_convs(blk: Bottleneck) -> List[nn.Conv2d]:
    return [blk.conv1, blk.conv2, blk.conv3] + ([blk.downsample[0]] if blk.downsample is not None else [])


def _stem(x: Tensor, stem) -> Tuple[Tensor, Tuple[int, int]]:
    """the stem and the max-pool: the image batch x -> layer 1's input token rows and map size"""
    _, _, H, W = x.shape
    hw = ((H - 1) // 2 + 1, (W - 1) // 2 + 1)
    t = cabi.maxpool3x3s2_tokens(cabi.resnet_stem(x, *stem), hw)
    return t, ((hw[0] - 1) // 2 + 1, (hw[1] - 1) // 2 + 1)


def _bottleneck(convs, t: Tensor, hw) -> Tuple[Tensor, Tuple[int, int]]:
    """one Bottleneck without autograd: (conv1, conv2, conv3, downsample or None) TokenConvs on the token rows t of an hw map
    -> the block's output rows and map size.  The residual is the downsample's fresh output, or a block input that only this
    block reads (an earlier block of the same stage): conv3 writes over it in place."""
    c1, c2, c3, ds = convs
    s = cabi.pow2_scale(t, 12)
    y1 = c1(t, hw, s)
    y2 = c2(y1, hw, cabi.pow2_scale(y1, 12))
    s2 = cabi.pow2_scale(y2, 12)
    ident = ds(t, hw, s) if ds is not None else t
    return c3(y2, c2.out_hw(hw), s2, out=ident, z=ident), c2.out_hw(hw)


class _TrainRun:
    """what _TrainBlocks needs beyond tensors: per block its TokenConvs, whether each of their weights trains (conv1, conv2,
    conv3, the downsample's if any) and the stage it ends (or None), the input map size"""

    def __init__(self, convs, trainable, ends, hw):
        self.convs, self.trainable, self.ends, self.hw = convs, trainable, ends, hw
        self.returned = [i for i in ends if i is not None]
        self.out_hw = {}


class _TrainBlocks(torch.autograd.Function):
    """The Bottlenecks from the first trainable one to the last kept stage, on token rows.  Inputs: the run, the token rows of
    the first block's input (no gradient), the trainable convolution weights in block order.  Outputs: the token rows of every
    stage that ends in the run.  The backward walks the chain once, G being the gradient at a block's pre-ReLU sum:
    wgrad3(G, y2); dy2 = dgrad3(G) * [y2 > 0]; wgrad2(dy2, y1); dy1 = dgrad2(dy2) * [y1 > 0]; wgrad1(dy1, t); and, when an
    earlier block needs it, G_prev = (dgrad1(dy1) + d_id) * [t > 0] with d_id = G or dgrad_ds(G) (+ the gradient of the
    returned map t, if it is one), each product and sum in a convolution's epilogue."""

    @staticmethod
    def forward(ctx, run: _TrainRun, t: Tensor, *weights: Tensor):
        hw = run.hw
        saved, outs = [], []
        for (c1, c2, c3, ds), end in zip(run.convs, run.ends):
            s = cabi.pow2_scale(t, 12)
            y1 = c1(t, hw, s)
            s1 = cabi.pow2_scale(y1, 12)
            y2 = c2(y1, hw, s1)
            s2 = cabi.pow2_scale(y2, 12)
            hw2 = c2.out_hw(hw)
            if ds is not None:
                ident = ds(t, hw, s)
                out = c3(y2, hw2, s2, out=ident, z=ident)
            else:
                out = c3(y2, hw2, s2, z=t)  # a fresh output: the block input is kept for the backward
            saved += [t, s, y1, s1, y2, s2]
            t, hw = out, hw2
            if end is not None:
                outs.append(t)
                run.out_hw[end] = hw
        ctx.run = run
        ctx.save_for_backward(*saved, t)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        run = ctx.run
        saved = ctx.saved_tensors
        # a returned map's gradient as token rows: a view when it came channels-last, else one copy
        ext = {end: g if g.is_contiguous() else g.contiguous() for end, g in zip(run.returned, grads)}
        dws = []
        nblk = len(run.convs)
        hws = [run.hw]
        for c1, c2, c3, ds in run.convs:
            hws.append(c2.out_hw(hws[-1]))
        # the deepest returned map's gradient, through the last block's ReLU
        G = torch.ops.aten.threshold_backward(ext[run.returned[-1]], saved[-1], 0)
        for j in range(nblk - 1, -1, -1):
            c1, c2, c3, ds = run.convs[j]
            tr = run.trainable[j]
            t, s, y1, s1, y2, s2 = saved[6 * j: 6 * j + 6]
            hw, hw2 = hws[j], hws[j + 1]
            need_in = j > 0
            gs = cabi.pow2_scale(G, 12)
            blk_dw = {}
            if tr[2]:
                blk_dw[3] = c3.wgrad(G, gs, y2, s2, hw2)
            if tr[1] or tr[0] or need_in:
                dy2 = c3.dgrad(G, hw2, gs, m=y2)
                s_dy2 = cabi.pow2_scale(dy2, 12)
                if tr[1]:
                    blk_dw[2] = c2.wgrad(dy2, s_dy2, y1, s1, hw)
                if tr[0] or need_in:
                    dy1 = c2.dgrad(dy2, hw, s_dy2, m=y1)
                    s_dy1 = cabi.pow2_scale(dy1, 12)
                    if tr[0]:
                        blk_dw[1] = c1.wgrad(dy1, s_dy1, t, s, hw)
            if ds is not None and tr[3]:
                blk_dw[4] = ds.wgrad(G, gs, t, s, hw)
            if need_in:
                z = ext.get(run.ends[j - 1]) if run.ends[j - 1] is not None else None
                if ds is not None:
                    d = ds.dgrad(G, hw, gs, z=z)
                else:
                    d = G if z is None else G + z
                G = c1.dgrad(dy1, hw, s_dy1, z=d, m=t, out=d)
            dws.append([blk_dw[i] for i in (1, 2, 3, 4) if i in blk_dw])
        return (None, None) + tuple(dw for blk in reversed(dws) for dw in blk)
