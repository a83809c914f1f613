"""ChannelMapper: the input neck between the backbone and the transformer (models/necks/channel_mapper.py:8-80 of the original
project), used by every shipped config (configs/salience_detr/*.py).

Same class name, constructor arguments, sub-module / parameter names (``convs.<i>.0`` the convolution, ``convs.<i>.1`` the
GroupNorm), initialisation and ``forward`` as the reference, so a reference ``state_dict`` loads with ``strict=True`` and a
detector checkpoint's ``neck.*`` keys load through ``load_reference_checkpoint(mapper, ckpt, prefix="neck.")``.  ``forward``
(an ``OrderedDict`` or dict of NCHW maps -> list of NCHW maps) is the reference's op chain in torch whenever ``tokens_supported``
does not hold: in training with autograd, on the CPU, and for configurations the kernels do not take.

``forward_tokens(inputs) -> (tokens (b, Nv, C), shapes_list)`` is the inference path (CUDA fp32, no autograd).  Every
convolution is ``sdetr_conv2d_f16x3`` (3xFP16 on wgmma, fp32-class accuracy whatever ``torch.backends.cudnn.allow_tf32`` says)
writing straight into its level slice of one token buffer; one ``sdetr_group_norm_tokens`` call then normalises all levels in
place.  Channels-last inputs are read in place as token rows; NCHW inputs are transposed once each
(``sdetr_token_map_transpose``).  No host synchronisation: the call can be captured in a CUDA graph.  When ``tokens_supported``
holds, ``forward`` returns the levels as NCHW *views* of that buffer (``level_views``): same values and shapes as the reference,
and ``SalienceTransformer`` recognises them (``tokens_of``) and takes the buffer as its tokens without a transpose.
"""
from __future__ import annotations

from functools import partial
from typing import List, Mapping, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import cabi, derived
from .neck import Conv2dNormActivation, TokenConv


# ---- the token-buffer view layout: both directions ----------------------------------------------------------------------
def level_views(tokens: Tensor, shapes: Sequence[Tuple[int, int]]) -> List[Tensor]:
    """(b, Nv, C) token buffer -> per-level (b, C, H, W) views with strides (Nv*C, 1, W*C, C), levels in token order."""
    views, s = [], 0
    for h, w in shapes:
        views.append(tokens[:, s:s + h * w].unflatten(1, (h, w)).permute(0, 3, 1, 2))
        s += h * w
    return views


def tokens_of(maps: Sequence[Tensor]) -> Optional[Tensor]:
    """The (b, Nv, C) token buffer whose ``level_views`` ``maps`` are (the levels tile it exactly, in order), else None."""
    maps = list(maps)
    if not maps or not all(torch.is_tensor(m) and m.dim() == 4 for m in maps):
        return None
    base = maps[0]
    b, c = base.shape[:2]
    nv = sum(m.shape[2] * m.shape[3] for m in maps)
    off, s = base.storage_offset(), 0
    for m in maps:
        h, w = m.shape[2:]
        if m.stride() != (nv * c, 1, w * c, c) or m.shape[:2] != (b, c) or m.storage_offset() != off + s * c:
            return None
        if m.dtype != base.dtype or m.device != base.device or m.untyped_storage().data_ptr() != base.untyped_storage().data_ptr():
            return None
        s += h * w
    if (off + b * nv * c) * base.element_size() > base.untyped_storage().nbytes():
        return None
    return base.as_strided((b, nv, c), (nv * c, c, 1), off)


# ---- the module --------------------------------------------------------------------------------------------------------
class ChannelMapper(nn.Module):
    def __init__(self, in_channels: List[int], out_channels: int, num_outs: int, kernel_size: int = 1, stride: int = 1,
                 groups: int = 1, norm_layer=partial(nn.GroupNorm, 32), activation_layer: nn.Module = None, dilation: int = 1,
                 inplace: bool = True, bias: bool = None):
        self.in_channels = in_channels
        super().__init__()
        self.convs = nn.ModuleList()
        self.num_channels = [out_channels] * num_outs
        for in_channel in in_channels:
            self.convs.append(Conv2dNormActivation(in_channels=in_channel, out_channels=out_channels, kernel_size=kernel_size,
                                                   stride=stride, padding=(kernel_size - 1) // 2, bias=bias, groups=groups,
                                                   dilation=dilation, norm_layer=norm_layer, activation_layer=activation_layer,
                                                   inplace=inplace))
        for _ in range(num_outs - len(in_channels)):
            self.convs.append(Conv2dNormActivation(in_channels=in_channel, out_channels=out_channels, kernel_size=3, stride=2,
                                                   padding=1, bias=bias, groups=groups, dilation=dilation, norm_layer=norm_layer,
                                                   activation_layer=activation_layer, inplace=inplace))
            in_channel = out_channels
        self.init_weights()

    def init_weights(self):
        for layer in self.modules():
            if isinstance(layer, nn.Conv2d):
                nn.init.xavier_uniform_(layer.weight, gain=1)
                if layer.bias:  # the reference's test: a no-op when the conv has no bias (the GroupNorm default)
                    nn.init.constant_(layer.bias, 0)

    def forward(self, inputs):
        values = list(inputs.values())
        if self.tokens_supported(values):
            return level_views(*self.forward_tokens(values))
        assert len(values) == len(self.in_channels)
        outs = [self.convs[i](values[i]) for i in range(len(values))]
        for i in range(len(values), len(self.convs)):
            if i == len(values):
                outs.append(self.convs[i](values[-1]))
            else:
                outs.append(self.convs[i](outs[-1]))
        return outs

    # ---- token-layout inference --------------------------------------------------------------------------------------
    def tokens_supported(self, inputs) -> bool:
        """True when forward_tokens can run this call: nothing needs a gradient (autograd off, or neither the inputs nor the
        parameters require one), CUDA fp32 inputs of the configured widths (channels-last ones 16-byte aligned), every conv
        with dilation 1 and in / groups and out / groups multiples of 64, the main convs 1x1 stride 1, every norm exactly
        nn.GroupNorm dividing the width (all with the same num_groups and eps), and no activation."""
        xs = list(inputs.values()) if isinstance(inputs, Mapping) else list(inputs)
        if len(xs) != len(self.in_channels) or len(xs) == 0:
            return False
        dev = xs[0].device
        for x, cin in zip(xs, self.in_channels):
            if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.device == dev):
                return False
            if x.shape[0] != xs[0].shape[0] or x.shape[1] != cin or x.shape[2] * x.shape[3] == 0:
                return False
            if x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16:
                return False
        if torch.is_grad_enabled() and (any(x.requires_grad for x in xs) or any(p.requires_grad for p in self.parameters())):
            return False
        return self.layers_supported()

    def layers_supported(self) -> bool:
        """The layer half of tokens_supported (it does not look at inputs or autograd)."""
        norms = []
        for i, m in enumerate(self.convs):
            conv = m[0]
            if conv.dilation != (1, 1) or (conv.in_channels // conv.groups) % 64 or (conv.out_channels // conv.groups) % 64:
                return False
            main = i < len(self.in_channels)
            if main and (conv.kernel_size != (1, 1) or conv.stride != (1, 1) or conv.padding != (0, 0)):
                return False
            if len(m) != 2 or type(m[1]) is not nn.GroupNorm or conv.out_channels % m[1].num_groups:
                return False  # no norm, another norm, or an activation
            norms.append((m[1].num_groups, m[1].eps))
        return len(set(norms)) == 1

    def _kernel_weights(self):
        """convolutions in kernel form and the (L, C) GroupNorm affine tables, rebuilt when any parameter changes"""
        def build():
            convs = [TokenConv(m[0].weight.detach().float(), m[0].bias.detach().float() if m[0].bias is not None else None,
                               m[0].groups, m[0].stride[0]) for m in self.convs]
            gn = [m[1] for m in self.convs]
            ones = torch.ones(gn[0].num_channels, device=self.convs[0][0].weight.device)
            gamma = torch.stack([n.weight.detach() if n.affine else ones for n in gn]).float().contiguous()
            beta = torch.stack([n.bias.detach() if n.affine else ones * 0 for n in gn]).float().contiguous()
            return convs, gamma, beta, gn[0].num_groups, gn[0].eps
        return derived.cached(self, "kernel_weights", list(self.parameters()), build)

    def launches_per_forward(self, nchw_inputs: Optional[int] = None) -> int:
        """library launches of one forward_tokens: one transpose per NCHW input (default: all inputs), per convolution 2
        (activation scale + convolution), 3 per GroupNorm call -- one call for the main levels and the first extra level,
        one more per further extra level (each reads the normalised output before it)"""
        n_in = len(self.in_channels)
        nchw = n_in if nchw_inputs is None else nchw_inputs
        return nchw + 2 * len(self.convs) + 3 * (1 + max(0, len(self.convs) - n_in - 1))

    @staticmethod
    def _token_rows(x: Tensor) -> Tensor:
        """(b, C, H, W) -> (b, H*W, C) token rows: a view of a channels-last map, a transposed copy of any other"""
        b, c, h, w = x.shape
        if x.is_contiguous(memory_format=torch.channels_last):
            return x.as_strided((b, h * w, c), (h * w * c, c, 1), x.storage_offset())
        return cabi.maps_to_tokens([x.contiguous()])

    def forward_tokens(self, inputs) -> Tuple[Tensor, List[Tuple[int, int]]]:
        """The mapper on ``inputs`` (OrderedDict / dict / sequence of NCHW maps) -> ((b, Nv, C) tokens with the levels in the
        reference's output order, [(H, W), ...]); same values as forward() in torch.  No host synchronisation."""
        xs = list(inputs.values()) if isinstance(inputs, Mapping) else list(inputs)
        if not self.tokens_supported(xs):
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported)")
        convs, gamma, beta, groups, eps = self._kernel_weights()
        n_in, n_out = len(xs), len(self.convs)
        b, c = xs[0].shape[0], self.convs[0][0].out_channels
        shapes = [tuple(int(v) for v in x.shape[2:]) for x in xs]
        for _ in range(n_out - n_in):
            h, w = shapes[-1]
            shapes.append(((h - 1) // 2 + 1, (w - 1) // 2 + 1))  # 3x3, stride 2, padding 1
        sizes = [h * w for h, w in shapes]
        starts = [sum(sizes[:i]) for i in range(n_out)]
        # chained extra levels read an earlier output: its activation scale is taken over the whole buffer, so start from zeros
        out = (torch.zeros if n_out - n_in > 1 else torch.empty)(b, sum(sizes), c, device=xs[0].device, dtype=torch.float32)
        level = [out[:, s:s + n] for s, n in zip(starts, sizes)]
        rows = [self._token_rows(x) for x in xs]
        for i in range(n_in):
            convs[i](rows[i], shapes[i], cabi.pow2_scale(rows[i], 12), out=level[i])
        if n_out > n_in:  # the first extra level reads the last input's token rows
            convs[n_in](rows[-1], shapes[n_in - 1], cabi.pow2_scale(rows[-1], 12), out=level[n_in])
        first = min(n_out, n_in + 1)
        cabi.group_norm_tokens_(out[:, :starts[first - 1] + sizes[first - 1]], sizes[:first], gamma[:first], beta[:first], groups,
                                eps)
        for i in range(n_in + 1, n_out):
            convs[i](level[i - 1], shapes[i - 1], cabi.pow2_scale(out, 12), out=level[i])
            cabi.group_norm_tokens_(level[i], sizes[i:i + 1], gamma[i:i + 1], beta[i:i + 1], groups, eps)
        return out, shapes
