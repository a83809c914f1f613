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

Under autograd (``training_tokens_supported``: no convolution bias, at most one extra level) ``forward_tokens`` trains in token
layout and returns the same tokens, bit for bit.  One autograd Function splits every weight in each call, writes the pre-norm
levels into a saved buffer and normalises them into a fresh one.  Its backward is ``sdetr_group_norm_tokens_backward`` (the input
gradient written over the saved buffer, dgamma and dbeta per level), then per level ``sdetr_conv2d_f16x3_wgrad`` and, for inputs
that need one, ``sdetr_conv2d_f16x3_dgrad``; the last input's gradient adds the extra level's stride-2 input gradient in the
epilogue.  A channels-last input gets a channels-last gradient (a view of token rows: ``ResNetBackbone``'s backward reads it in
place), an NCHW input one transpose.  ``forward()`` stays the torch chain in training: callers opt in with
``mapper.forward_tokens(backbone.forward_tokens(images))``.  No host synchronisation and a fixed launch count
(``launches_per_training_step``), so a forward + backward can be captured in a CUDA graph.
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
        xs = _values(inputs)
        if not self._inputs_ok(xs) or self._autograd_records(xs):
            return False
        return self.layers_supported()

    def _inputs_ok(self, xs: List[Tensor]) -> bool:
        """one CUDA fp32 (b, C_i, H_i, W_i) map per input width on one device, none empty, channels-last ones 16-byte aligned"""
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
        return True

    def _autograd_records(self, xs: List[Tensor]) -> bool:
        return torch.is_grad_enabled() and (any(x.requires_grad for x in xs) or any(p.requires_grad for p in self.parameters()))

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

    def training_tokens_supported(self, inputs) -> bool:
        """True when forward_tokens trains this call in token layout: layers_supported(), the inputs tokens_supported asks for,
        every parameter fp32 on their device, autograd recording (grad enabled and some input or parameter requiring a
        gradient), no convolution bias and at most one extra level (chained extra levels need forward())."""
        xs = _values(inputs)
        if not self._inputs_ok(xs) or not self._autograd_records(xs):
            return False
        if any(p.device != xs[0].device or p.dtype != torch.float32 for p in self.parameters()):
            return False
        if any(m[0].bias is not None for m in self.convs) or len(self.convs) - len(self.in_channels) > 1:
            return False
        return self.layers_supported()

    def launches_per_training_step(self, inputs) -> int:
        """library launches of one forward_tokens under autograd on ``inputs`` and its backward (training_tokens_supported), from
        their layouts and which tensors require a gradient (no host synchronisation).  Forward: one transpose per NCHW input,
        one activation scale per input, per convolution 3 (weight scale, split, convolution), 3 for the GroupNorm.  Backward:
        5 for the GroupNorm gradient (+1 when a GroupNorm parameter trains), the scale of its result when a convolution needs
        it, 2 per trainable convolution weight, 1 per input gradient of a convolution, 1 transpose per NCHW input gradient."""
        xs = _values(inputs)
        n_in, n_conv = len(xs), len(self.convs)
        nchw = [not x.is_contiguous(memory_format=torch.channels_last) for x in xs]
        n = sum(nchw) + n_in + 3 * n_conv + 3 + 5
        gn = [p for m in self.convs for p in m[1].parameters()]
        n += any(p.requires_grad for p in gn)
        wg = [m[0].weight.requires_grad for m in self.convs]
        dg = [x.requires_grad for x in xs] + [xs[-1].requires_grad] * (n_conv - n_in)
        n += 2 * sum(wg) + sum(dg) + sum(r and c for r, c in zip((x.requires_grad for x in xs), nchw))
        return n + (any(wg) or any(dg))

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

    def _levels(self, xs: List[Tensor]):
        """([(H, W)] of every output level, their token counts, their first tokens)"""
        shapes = [tuple(int(v) for v in x.shape[2:]) for x in xs]
        for _ in range(len(self.convs) - len(xs)):
            h, w = shapes[-1]
            shapes.append(((h - 1) // 2 + 1, (w - 1) // 2 + 1))  # 3x3, stride 2, padding 1
        sizes = [h * w for h, w in shapes]
        return shapes, sizes, [sum(sizes[:i]) for i in range(len(sizes))]

    def _train_tokens(self, xs: List[Tensor]) -> Tuple[Tensor, List[Tuple[int, int]]]:
        """forward_tokens under autograd (training_tokens_supported): one _TrainMapper call"""
        shapes, sizes, _ = self._levels(xs)
        gn = [m[1] for m in self.convs]
        affine = gn[0].affine
        params = [m[0].weight for m in self.convs] + ([n.weight for n in gn] + [n.bias for n in gn] if affine else [])
        run = _TrainRun(self, shapes, sizes, affine)
        return _TrainMapper.apply(run, *xs, *params), shapes

    def forward_tokens(self, inputs) -> Tuple[Tensor, List[Tuple[int, int]]]:
        """The mapper on ``inputs`` (OrderedDict / dict / sequence of NCHW maps) -> ((b, Nv, C) tokens with the levels in the
        reference's output order, [(H, W), ...]); same values as forward() in torch.  No host synchronisation.  Under autograd
        (training_tokens_supported) the same tokens, bit for bit, with a token-layout backward."""
        xs = _values(inputs)
        if not self.tokens_supported(xs):
            if self.training_tokens_supported(xs):
                return self._train_tokens(xs)
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported / training_tokens_supported)")
        convs, gamma, beta, groups, eps = self._kernel_weights()
        n_in, n_out = len(xs), len(self.convs)
        b, c = xs[0].shape[0], self.convs[0][0].out_channels
        shapes, sizes, starts = self._levels(xs)
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


def _values(inputs) -> List[Tensor]:
    return list(inputs.values()) if isinstance(inputs, Mapping) else list(inputs)


class _TrainRun:
    """what _TrainMapper needs beyond tensors: the mapper's layout (inputs, convolutions, GroupNorm groups and eps), the level
    shapes and token counts, and whether the GroupNorms are affine (their weights and biases are then inputs too)"""

    def __init__(self, mapper: ChannelMapper, shapes, sizes, affine: bool):
        self.n_in, self.n_conv = len(mapper.in_channels), len(mapper.convs)
        self.groups = [m[0].groups for m in mapper.convs]
        self.strides = [m[0].stride[0] for m in mapper.convs]
        self.num_groups, self.eps = mapper.convs[0][1].num_groups, mapper.convs[0][1].eps
        self.shapes, self.sizes, self.affine = shapes, sizes, affine


class _TrainMapper(torch.autograd.Function):
    """The mapper with at most one extra level on token rows.  Inputs: the run, the input maps, the convolution weights, then
    (affine GroupNorms) the GroupNorm weights and biases.  Output: the (b, Nv, C) tokens of forward_tokens, bit-identical to
    the inference path.  The forward keeps the pre-norm tokens P; the backward writes the GroupNorm's input gradient over P, then
    per level the weight gradient and, for inputs that need one, the input gradient (the last input's main and extra-level
    gradients summed in the second convolution's epilogue)."""

    @staticmethod
    def forward(ctx, run: _TrainRun, *args):
        n_in, n_conv = run.n_in, run.n_conv
        xs, weights = args[:n_in], args[n_in:n_in + n_conv]
        need_x = ctx.needs_input_grad[1:1 + n_in]
        b, c, dev = xs[0].shape[0], weights[0].shape[0], xs[0].device
        if run.affine:
            gamma = torch.stack(args[n_in + n_conv:n_in + 2 * n_conv]).contiguous()
            beta = torch.stack(args[n_in + 2 * n_conv:]).contiguous()
        else:
            gamma = torch.ones(n_conv, c, device=dev, dtype=torch.float32)
            beta = torch.zeros(n_conv, c, device=dev, dtype=torch.float32)
        # split inside every call: an optimizer step between CUDA-graph replays changes the weights in place
        convs = [TokenConv(w.detach(), None, run.groups[i], run.strides[i], dgrad=need_x[min(i, n_in - 1)])
                 for i, w in enumerate(weights)]
        rows = [ChannelMapper._token_rows(x) for x in xs]
        scales = [cabi.pow2_scale(r, 12) for r in rows]
        P = torch.empty(b, sum(run.sizes), c, device=dev, dtype=torch.float32)
        level = _level_slices(P, run.sizes)
        for i in range(n_conv):
            j = min(i, n_in - 1)  # the extra level reads the last input
            convs[i](rows[j], run.shapes[j], scales[j], out=level[i])
        Y = cabi.group_norm_tokens_(P, run.sizes, gamma, beta, run.num_groups, run.eps, out=torch.empty_like(P))
        for conv in convs:
            conv.w_hi = conv.w_lo = None  # the backward reads only the input-gradient pairs
        ctx.run, ctx.convs, ctx.consumed = run, convs, False
        ctx.channels_last = [x.is_contiguous(memory_format=torch.channels_last) for x in xs]
        ctx.save_for_backward(P, gamma, *rows, *scales)
        return Y

    @staticmethod
    def backward(ctx, gY):
        run = ctx.run
        if ctx.consumed:
            raise RuntimeError("ChannelMapper.forward_tokens: the backward overwrites its saved tokens and runs once per forward")
        ctx.consumed = True
        n_in, n_conv = run.n_in, run.n_conv
        P, gamma, *rest = ctx.saved_tensors
        rows, scales = rest[:n_in], rest[n_in:]
        need = ctx.needs_input_grad[1:]
        need_x, need_w = need[:n_in], need[n_in:n_in + n_conv]
        need_gn = need[n_in + n_conv:] if run.affine else (False,) * (2 * n_conv)
        gY = gY.contiguous()
        dP, dgamma, dbeta = cabi.group_norm_tokens_backward(gY, P, run.sizes, gamma, run.num_groups, run.eps, dx=P,
                                                            dgamma=any(need_gn[:n_conv]), dbeta=any(need_gn[n_conv:]))
        level = _level_slices(dP, run.sizes)
        dw = [None] * n_conv
        dx = [None] * n_in
        if any(need_w) or any(need_x):
            gs = cabi.pow2_scale(dP, 12)
            for i, conv in enumerate(ctx.convs):
                j = min(i, n_in - 1)
                if need_w[i]:
                    dw[i] = conv.wgrad(level[i], gs, rows[j], scales[j], run.shapes[j])
            for j in range(n_in):
                if not need_x[j]:
                    continue
                z = None
                if j == n_in - 1 and n_conv > n_in:  # the extra level's stride-2 gradient, added in the main one's epilogue
                    z = ctx.convs[n_in].dgrad(level[n_in], run.shapes[j], gs)
                dx[j] = ctx.convs[j].dgrad(level[j], run.shapes[j], gs, z=z, out=z)
        grads_x = []
        for j, d in enumerate(dx):
            if d is None:
                grads_x.append(None)
                continue
            (h, w), cin = run.shapes[j], d.shape[2]
            if ctx.channels_last[j]:  # the input's layout: its token rows viewed as NCHW, no copy
                grads_x.append(d.view(d.shape[0], h, w, cin).permute(0, 3, 1, 2))
            else:
                grads_x.append(cabi.tokens_to_maps(d, [(h, w)])[0])
        grads_gn = ()
        if run.affine:
            grads_gn = tuple(dgamma[l] if need_gn[l] else None for l in range(n_conv)) + \
                tuple(dbeta[l] if need_gn[n_conv + l] else None for l in range(n_conv))
        return (None, *grads_x, *dw, *grads_gn)


def _level_slices(t: Tensor, sizes) -> List[Tensor]:
    out, s = [], 0
    for n in sizes:
        out.append(t[:, s:s + n])
        s += n
    return out
