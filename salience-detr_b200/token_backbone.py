"""What the token-layout backbones (backbone.py, convnext.py, swin.py) share around their kernels: weight loading, freezing,
the layer-independent half of ``tokens_supported``, the channels-last views of the returned token buffers, and
``FeatureBackbone``, the body of the backbones laid out as ``features``.  ResNetBackbone keeps the reference's named-attribute
layout (``conv1``, ``bn1``, ``layer1`` ...) and uses the module-level helpers only.
"""
from __future__ import annotations

from collections.abc import Mapping
from typing import Callable, Dict, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import cabi, derived


def load_weights(net: nn.Module, weights, skip_prefixes: Tuple[str, ...], who: str) -> None:
    """None: keep the initialisation.  A state dict (or one under "model"), or a local path read with torch.load: every key but
    those starting with one of ``skip_prefixes`` (the classifier) must match ``net`` exactly.  ``who`` names the backbone in
    the messages."""
    if weights is None:
        return
    if isinstance(weights, str):
        if weights.startswith(("http://", "https://")):
            raise RuntimeError(f"{who}: downloading weights is not supported ({weights}); pass a state dict or a local file")
        weights = torch.load(weights, map_location="cpu")
    if not isinstance(weights, Mapping):
        raise TypeError(f"{who}: weights must be None, a state dict or a path, got {type(weights).__name__}")
    if "model" in weights:
        weights = weights["model"]
    res = net.load_state_dict({k: v for k, v in weights.items() if not k.startswith(skip_prefixes)}, strict=False)
    missing = [k for k in res.missing_keys if not k.startswith(skip_prefixes)]
    if missing or res.unexpected_keys:
        raise RuntimeError(f"{who}: weights do not match the network: missing {missing}, unexpected {res.unexpected_keys}")


def freeze(modules: Sequence[nn.Module]) -> None:
    """eval() and no gradient for every parameter of each module"""
    for m in modules:
        m.eval()
        for p in m.parameters():
            p.requires_grad = False


def cuda_image(x) -> bool:
    """a non-empty NCHW-contiguous CUDA fp32 (b, 3, H, W) tensor"""
    return (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.numel() > 0
            and x.is_contiguous())


def on_device_fp32(module: nn.Module, device: torch.device) -> bool:
    """every parameter fp32 on ``device``, every buffer on ``device`` and fp32 if it is floating point (an integer index
    buffer such as Swin's relative_position_index stays integer)"""
    if any(p.device != device or p.dtype != torch.float32 for p in module.parameters()):
        return False
    return all(t.device == device and (t.dtype == torch.float32 or not t.is_floating_point()) for t in module.buffers())


def tokens_ready(module: nn.Module, x) -> bool:
    """The layer-independent half of tokens_supported: ``x`` a cuda_image, the module on_device_fp32 on its device, and nothing
    that needs a gradient (autograd off, or neither the input nor a parameter requires one)."""
    if not cuda_image(x) or not on_device_fp32(module, x.device):
        return False
    return not (torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in module.parameters())))


def token_maps(feats, return_indices: Sequence[int], name_of: Callable[[int], str]) -> Dict[str, Tensor]:
    """{name_of(i): map} for i in return_indices, feats[i] being a (b, h*w, C) token buffer and its (h, w): each map the
    channels-last (b, C, h, w) view of its buffer, strides (h*w*C, 1, w*C, C)"""
    outs = {}
    for i in return_indices:
        t, (h, w) = feats[i]
        outs[name_of(i)] = t.unflatten(1, (h, w)).permute(0, 3, 1, 2)
    return outs


class FeatureBackbone(nn.Module):
    """A backbone whose ``features`` are stem, stage, downsample, stage, ... of ``network``, truncated after the last returned
    stage.  A subclass sets ``model_arch`` (name -> ``network`` arguments), ``network``, ``skip_prefixes`` (the classifier's
    keys, ignored in loaded weights) and ``kblock`` / ``kdown`` (a block and a downsample in kernel form), and defines
    ``_config(arch, kwargs)`` (the ``network`` arguments with the keyword arguments merged in), ``_stage_channels(cfg, i)``,
    ``tokens_supported``, ``layers_supported``, ``launches_per_forward``, and ``_block_tokens(k, t, hw)`` /
    ``_down_tokens(k, t, hw)`` (one block / downsample in kernel form on the token rows t of an hw map -> the output rows)
    with ``_down_hw(hw)``, the map size after a downsample."""

    def __init__(self, arch: str, weights=None, return_indices: Tuple[int, ...] = (0, 1, 2, 3), freeze_indices: Tuple = (),
                 **kwargs):
        super().__init__()
        if arch not in self.model_arch:
            raise ValueError(f"Expected architecture in {list(self.model_arch)} but got {arch}")
        cfg = self._config(arch, kwargs)
        net = self.network(**cfg)
        load_weights(net, weights, self.skip_prefixes, type(self).__name__)
        feats = net.features
        if len(freeze_indices) > 0:
            freeze([feats[0]] + [feats[j] for i in freeze_indices for j in (2 * i + 1, 2 * i + 2) if j < len(feats)])
        self.return_indices = tuple(int(i) for i in return_indices)
        # the modules the feature extractor keeps: the stem and everything up to the last returned stage
        self.features = nn.Sequential(*list(feats)[:2 * max(self.return_indices) + 2])
        self.num_channels = [self._stage_channels(cfg, i) for i in self.return_indices]

    def _num_stages(self) -> int:
        return max(self.return_indices) + 1

    def forward(self, x: Tensor) -> Dict[str, Tensor]:
        if self.tokens_supported(x):
            return self.forward_tokens(x)
        return self.forward_torch(x)

    def forward_torch(self, x: Tensor) -> Dict[str, Tensor]:
        """the reference's op chain in torch: {"features.{2i+1}": map} for i in return_indices"""
        feats = {}
        x = self.features[0](x)
        for i in range(self._num_stages()):
            x = self.features[2 * i + 1](x)
            feats[i] = x
            if i + 1 < self._num_stages():
                x = self.features[2 * i + 2](x)
        return {f"features.{2 * i + 1}": self._nchw(feats[i]) for i in self.return_indices}

    @staticmethod
    def _nchw(x: Tensor) -> Tensor:
        """a stage's output as the reference returns it"""
        return x

    def _kernel_weights(self):
        """the stem ((48, C) weight, bias, LayerNorm weight, bias, eps) and per kept stage its blocks and the downsample after
        it (None after the last), rebuilt when any parameter or buffer changes"""
        def build():
            conv, ln = self.features[0][0], self.features[0][-1]
            c = conv.out_channels
            stem = (conv.weight.detach().reshape(c, 48).t().contiguous(), conv.bias.detach(), ln.weight.detach(),
                    ln.bias.detach(), ln.eps)
            stages = []
            for i in range(self._num_stages()):
                blocks = [self.kblock(blk) for blk in self.features[2 * i + 1]]
                stages.append((blocks, self.kdown(self.features[2 * i + 2]) if i + 1 < self._num_stages() else None))
            return stem, stages
        return derived.cached(self, "kernel_weights", list(self.parameters()) + list(self.buffers()), build)

    def forward_tokens(self, x: Tensor) -> Dict[str, Tensor]:
        """The backbone on ``x`` (b, 3, H, W) -> {"features.{2i+1}": (b, C, h, w)} for i in return_indices, each a channels-last
        view (strides (h*w*C, 1, w*C, C)) of its own (b, h*w, C) token buffer; the values of forward() in torch.  No host
        synchronisation."""
        if not self.tokens_supported(x):
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported)")
        (stem_w, stem_b, ln_w, ln_b, eps), stages = self._kernel_weights()
        hw = (x.shape[2] // 4, x.shape[3] // 4)
        t = cabi.convnext_stem(x, stem_w, stem_b, ln_w, ln_b, eps)
        feats = []
        for blocks, ds in stages:
            for k in blocks:
                t = self._block_tokens(k, t, hw)
            feats.append((t, hw))
            if ds is not None:
                t = self._down_tokens(ds, t, hw)
                hw = self._down_hw(hw)
        return token_maps(feats, self.return_indices, lambda i: f"features.{2 * i + 1}")
