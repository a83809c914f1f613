"""RepVGG-PluX neck between the encoder and the decoder (models/necks/repnet.py:125-245 of the original project).

Same class names, constructor arguments, sub-module / parameter / buffer names and ``forward`` as the reference, so a released
checkpoint's ``transformer.neck.*`` keys load with ``strict=True``.  ``forward`` (an ``OrderedDict`` of NCHW maps) is the
reference's op chain in torch: it is what runs in training (BatchNorm with batch statistics, and
``nn.SyncBatchNorm.convert_sync_batchnorm`` works on it), on the CPU, and for widths the kernels do not take.

``RepVGGPluXNetwork.forward_tokens(memory, shapes_list)`` is the inference path: eval mode, CUDA, no autograd.  It reads the
encoder memory's level slices in place and writes every level straight into a fresh ``(b, Nv, C)`` tensor, with no NCHW copy
either way.  Per parameter / buffer version the eval weights are folded once and cached: every BatchNorm into its convolution,
each RepVGG block's ``conv1 (3x3) + alpha * conv2 (1x1)`` into one grouped 3x3 convolution (the 1x1 in the centre tap), and each
CSP layer's ``conv1 || conv2`` (two 1x1 over the same input) into one projection.  The kernels (``include/sdetr_b200.h``):
``sdetr_conv2d_f16x3`` (implicit-GEMM convolution, 3xFP16 on wgmma, bias + SiLU epilogue), ``sdetr_context_gate``
(SqueezeAndExcitation + the block's residual) and ``sdetr_upsample_nearest_concat`` (the top-down path's operand).
``TokenConv`` is the convolution in kernel form, which the ChannelMapper and the ResNet backbone use too.

In training, or whenever autograd records (``training_tokens_supported``), ``forward_tokens`` follows the reference's op
structure instead of the folded one: every convolution (a RepVGG block's 3x3 and 1x1, a CSP layer's conv1 and conv2 apart) runs
on the same kernel through an autograd Function.  Its forward splits the weight once (``sdetr_conv2d_f16x3_split_weight``) into
both fp16 layouts; its backward is the input gradient (``sdetr_conv2d_f16x3_dgrad`` with the flipped, per-group transposed
weights) and the weight gradient (``sdetr_conv2d_f16x3_wgrad``).  Each
BatchNorm is the module itself on the channels-last ``(b, C, H, W)`` view of the token rows (no copy), so batch statistics, running statistics,
``momentum``, eval mode with gradients and ``nn.SyncBatchNorm`` behave as the modules define.  SiLU, the context gate, the
residuals and the concatenations are torch ops on token rows; the top-down operand's backward is
``sdetr_upsample_nearest_concat_backward``.  No host synchronisation and a fixed launch count, so a forward + backward can be
captured in a CUDA graph.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Callable, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn
from torch.nn import functional as F

from . import cabi, derived


class Conv2dNormActivation(nn.Sequential):
    """Conv2d (index 0), optional norm (1) and optional activation (2) -- models/bricks/misc.py:62-160."""

    def __init__(self, in_channels: int, out_channels: int, kernel_size: int = 3, stride: int = 1, padding: Optional[int] = None,
                 groups: int = 1, norm_layer: Optional[Callable[..., nn.Module]] = nn.BatchNorm2d,
                 activation_layer: Optional[Callable[..., nn.Module]] = nn.ReLU, dilation: int = 1,
                 inplace: Optional[bool] = True, bias: Optional[bool] = None) -> None:
        if padding is None:
            padding = (kernel_size - 1) // 2 * dilation
        if bias is None:
            bias = norm_layer is None
        layers = [nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, dilation=dilation, groups=groups, bias=bias)]
        if norm_layer is not None:
            layers.append(norm_layer(out_channels))
        if activation_layer is not None:
            layers.append(activation_layer(**({} if inplace is None else {"inplace": inplace})))
        super().__init__(*layers)
        self.out_channels = out_channels


class SqueezeAndExcitation(nn.Module):
    """GCNet-style context gate (models/bricks/basic.py:29-54): conv_mask -> softmax over all H*W pixels -> weighted sum of the
    pixels -> C -> C/r -> C -> sigmoid, multiplied into x."""

    def __init__(self, channels, reduction=16):
        super().__init__()
        self.conv_mask = nn.Conv2d(channels, 1, kernel_size=1)
        self.softmax = nn.Softmax(dim=2)
        self.se_module = nn.Sequential(
            nn.Conv2d(channels, channels // reduction, kernel_size=1, stride=1, bias=False),
            nn.ReLU(inplace=True),
            nn.Conv2d(channels // reduction, channels, kernel_size=1, stride=1, bias=False),
            nn.Sigmoid(),
        )
        nn.init.kaiming_normal_(self.conv_mask.weight, mode="fan_in", nonlinearity="relu")

    def forward(self, x):
        batch, channel, height, width = x.shape
        input_x = x.view(batch, channel, height * width).unsqueeze(1)
        context_mask = self.softmax(self.conv_mask(x).view(batch, 1, height * width)).unsqueeze(-1)
        context = torch.matmul(input_x, context_mask).view(batch, channel, 1, 1)
        return self.se_module(context) * x


class RepVggPluXBlock(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, activation_layer: nn.Module = nn.ReLU, inplace: bool = True,
                 groups: int = 4, alpha: bool = False):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.activation = activation_layer(inplace=True)
        self.conv1 = Conv2dNormActivation(in_channels, out_channels, kernel_size=3, stride=1, padding=1, groups=groups,
                                          activation_layer=None, inplace=inplace)
        self.conv2 = Conv2dNormActivation(in_channels, out_channels, kernel_size=1, stride=1, padding=0, groups=groups,
                                          activation_layer=None, inplace=inplace)
        self.alpha = nn.Parameter(torch.tensor(1.0)) if alpha else 1.0
        self.se_module = SqueezeAndExcitation(channels=out_channels)
        self.identity = nn.Conv2d(in_channels, out_channels, kernel_size=1) if in_channels != out_channels else nn.Identity()

    def forward(self, x: Tensor) -> Tensor:
        y = self.conv1(x) + self.alpha * self.conv2(x)
        y = self.se_module(self.activation(y))
        return y + self.identity(x)


class CSPRepPluXLayer(nn.Module):
    def __init__(self, in_channels: int, out_channels: int, num_blocks: int = 3, expansion: float = 1.0, groups: int = 4,
                 norm_layer: nn.Module = nn.BatchNorm2d, activation_layer: nn.Module = nn.SiLU):
        super().__init__()
        hidden_channels = int(out_channels * expansion)
        self.conv1 = Conv2dNormActivation(in_channels, hidden_channels, kernel_size=1, stride=1, norm_layer=norm_layer,
                                          activation_layer=activation_layer, inplace=True)
        self.conv2 = Conv2dNormActivation(in_channels, hidden_channels, kernel_size=1, stride=1, norm_layer=norm_layer,
                                          activation_layer=activation_layer, inplace=True)
        self.bottlenecks = nn.Sequential(*[RepVggPluXBlock(hidden_channels, hidden_channels, groups=groups,
                                                           activation_layer=activation_layer) for _ in range(num_blocks)])
        if hidden_channels != out_channels:
            self.conv3 = Conv2dNormActivation(hidden_channels, out_channels, kernel_size=1, stride=1, norm_layer=norm_layer,
                                              activation_layer=activation_layer)
        else:
            self.conv3 = nn.Identity()

    def forward(self, x: Tensor) -> Tensor:
        x = self.bottlenecks(self.conv1(x)) + self.conv2(x)
        return self.conv3(x)


# ---- eval-weight folding ------------------------------------------------------------------------------------------------
def fold_conv_norm(m: Conv2dNormActivation, dtype=None) -> Tuple[Tensor, Tensor]:
    """(weight, bias) of the conv with its BatchNorm (eval statistics) folded in: w * g / sqrt(var + eps), (b - mean) * g /
    sqrt(var + eps) + beta.  ``dtype``: arithmetic type (default: the parameters')."""
    conv = m[0]
    dtype = dtype or conv.weight.dtype
    w = conv.weight.detach().to(dtype)
    b = conv.bias.detach().to(dtype) if conv.bias is not None else torch.zeros(w.shape[0], dtype=dtype, device=w.device)
    if len(m) > 1 and isinstance(m[1], nn.BatchNorm2d):
        bn = m[1]
        s = bn.weight.detach().to(dtype) / torch.sqrt(bn.running_var.detach().to(dtype) + bn.eps)
        w = w * s.view(-1, 1, 1, 1)
        b = (b - bn.running_mean.detach().to(dtype)) * s + bn.bias.detach().to(dtype)
    return w, b


def fold_repvgg(blk: RepVggPluXBlock, dtype=None) -> Tuple[Tensor, Tensor]:
    """conv1 (3x3) + alpha * conv2 (1x1) of a block as one 3x3 convolution: the 1x1 goes into the centre tap."""
    w1, b1 = fold_conv_norm(blk.conv1, dtype)
    w2, b2 = fold_conv_norm(blk.conv2, dtype)
    alpha = blk.alpha.detach().to(w1.dtype) if isinstance(blk.alpha, Tensor) else blk.alpha
    w = w1.clone()
    w[:, :, 1, 1] += alpha * w2[:, :, 0, 0]
    return w, b1 + alpha * b2


def fold_csp_projection(layer: CSPRepPluXLayer, dtype=None) -> Tuple[Tensor, Tensor]:
    """conv1 || conv2 of a CSP layer (both 1x1 over the same input) as one projection with 2 * hidden outputs."""
    w1, b1 = fold_conv_norm(layer.conv1, dtype)
    w2, b2 = fold_conv_norm(layer.conv2, dtype)
    return torch.cat([w1, w2], 0), torch.cat([b1, b2], 0)


def nearest_index(n_in: int, n_out: int) -> Tensor:
    """Source index of each output position of torch's ``F.interpolate(mode="nearest")`` along one axis:
    min(floor(dst * (float)in / out), in - 1) in fp32 -- the rule sdetr_upsample_nearest_concat computes."""
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    src = torch.floor(torch.arange(n_out, dtype=torch.float32) * scale).to(torch.int64)
    return src.clamp(max=n_in - 1)


def nearest_ranges(n_in: int, n_out: int) -> Tuple[Tensor, Tensor]:
    """[begin, end) of the output positions that read each input position under nearest_index: the ranges the upsample
    backward (sdetr_upsample_nearest_concat_backward) sums over"""
    src = nearest_index(n_in, n_out)
    s = torch.arange(n_in, dtype=torch.int64)
    return torch.searchsorted(src, s, right=False), torch.searchsorted(src, s, right=True)


class TokenConv:
    """One convolution on token rows (sdetr_conv2d_f16x3 and its gradients), padding k / 2.  Built from an fp32 (Cout, Cin /
    groups, k, k) weight, split here (conv2d_f16x3_split_weight) into the forward's fp16 pair and, with ``dgrad``, the input
    gradient's; ``bias``: fp32 (Cout) or None; ``act``: 0, cabi.ACT_RELU or cabi.ACT_SILU; ``bn_scale``: an optional (Cout)
    factor of the weight gradient (a FrozenBatchNorm scale folded into the weight).  The caller passes each activation scale
    (cabi.pow2_scale, target 12), so convolutions that read the same tensor share one."""

    def __init__(self, w: Tensor, bias: Optional[Tensor], groups: int = 1, stride: int = 1, act: int = 0, dgrad: bool = False,
                 bn_scale: Optional[Tensor] = None):
        self.shape, self.groups, self.stride, self.act = tuple(w.shape), groups, stride, act
        self.w_hi, self.w_lo, self.d_hi, self.d_lo, self.w_scale = cabi.conv2d_f16x3_split_weight(w.contiguous(), groups, dgrad)
        self.bias, self.bn_scale = bias, bn_scale

    def out_hw(self, hw):
        k = self.shape[-1]
        return tuple((v + 2 * (k // 2) - k) // self.stride + 1 for v in hw)

    def __call__(self, x: Tensor, hw, a_scale: Tensor, out=None, z=None) -> Tensor:
        """act(conv(x) + bias (+ z)): x (b, H*W, Cin) view of an (H, W) = hw map; out, z: optional (b, Ho*Wo, Cout) views"""
        return cabi.conv2d_f16x3(x, hw, a_scale, self.w_hi, self.w_lo, self.w_scale, self.bias, self.groups, self.shape[-1],
                                 self.stride, self.act, out=out, z=z)

    def dgrad(self, g: Tensor, hw, g_scale: Tensor, z=None, m=None, out=None) -> Tensor:
        """the input gradient (+ z, then 0 where m <= 0) of the (H, W) = hw map from g (b, Ho*Wo, Cout)"""
        return cabi.conv2d_f16x3_dgrad(g, self.out_hw(hw), g_scale, self.d_hi, self.d_lo, self.w_scale, self.groups,
                                       self.shape[-1], self.stride, hw, z=z, m=m, out=out)

    def wgrad(self, g: Tensor, g_scale: Tensor, x: Tensor, x_scale: Tensor, hw) -> Tensor:
        """the weight gradient (times bn_scale) from g (b, Ho*Wo, Cout) and the input x of the (H, W) = hw map"""
        return cabi.conv2d_f16x3_wgrad(g, g_scale, x, x_scale, hw, self.shape, self.stride, cout_scale=self.bn_scale)


class _TokenConv2d(torch.autograd.Function):
    """y = conv2d(x, weight) on token rows, no bias (every convolution of the training path is followed by a BatchNorm).
    x: (b, H*W, Cin) view; a_scale: pow2_scale (target 12) of a contiguous tensor that holds x, shared by the convolutions that
    read the same input.  The weight is split once per call into both fp16 layouts the forward and the input gradient read."""

    @staticmethod
    def forward(ctx, x, weight, a_scale, hw, stride):
        conv = TokenConv(weight.detach(), None, x.shape[2] // weight.shape[1], stride, dgrad=ctx.needs_input_grad[0])
        y = conv(x, hw, a_scale)
        conv.w_hi = conv.w_lo = None  # the backward reads only the input-gradient pair
        ctx.save_for_backward(x, a_scale)
        ctx.conv, ctx.hw = conv, hw
        return y

    @staticmethod
    def backward(ctx, gy):
        x, a_scale = ctx.saved_tensors
        gy = gy.contiguous()  # the BatchNorm gradients this path produces already are: no copy
        g_scale = cabi.pow2_scale(gy, 12)
        dx = ctx.conv.dgrad(gy, ctx.hw, g_scale) if ctx.needs_input_grad[0] else None
        dw = ctx.conv.wgrad(gy, g_scale, x, a_scale, ctx.hw) if ctx.needs_input_grad[1] else None
        return dx, dw, None, None, None


class _UpsampleConcat(torch.autograd.Function):
    """[nearest(hi) | lo] on token rows (sdetr_upsample_nearest_concat) with its backward"""

    @staticmethod
    def forward(ctx, hi, hi_hw, lo, lo_hw):
        ctx.hi_hw, ctx.lo_hw, ctx.c = hi_hw, lo_hw, hi.shape[2]
        return cabi.upsample_nearest_concat(hi, hi_hw, lo, lo_hw)

    @staticmethod
    def backward(ctx, g):
        c = ctx.c
        d_hi = cabi.upsample_nearest_concat_backward(g[:, :, :c], ctx.lo_hw, ctx.hi_hw) if ctx.needs_input_grad[0] else None
        return d_hi, None, g[:, :, c:], None


def _norm_rows(bn: nn.Module, y: Tensor, hw) -> Tensor:
    """the BatchNorm module on (b, H*W, C) token rows, which are the channels-last layout of (b, C, H, W): torch's
    channels-last BatchNorm reads them in place (an (N, C, 1, 1) view would take the NCHW kernels with one pixel per image)"""
    b, n, c = y.shape
    return bn(y.view(b, hw[0], hw[1], c).permute(0, 3, 1, 2)).permute(0, 2, 3, 1).reshape(b, n, c)


def _gate_rows(se: SqueezeAndExcitation, y: Tensor) -> Tensor:
    """SqueezeAndExcitation on (b, HW, C) token rows"""
    c = y.shape[2]
    p = torch.softmax(F.linear(y, se.conv_mask.weight.view(1, c), se.conv_mask.bias).squeeze(2), 1)
    ctx = torch.bmm(p.unsqueeze(1), y).squeeze(1)
    gate = torch.sigmoid(F.linear(F.relu(F.linear(ctx, se.se_module[0].weight.view(-1, c))), se.se_module[2].weight.view(c, -1)))
    return gate.unsqueeze(1) * y


class _KGate:
    def __init__(self, se: SqueezeAndExcitation):
        c = se.conv_mask.weight.shape[1]
        self.w_mask = se.conv_mask.weight.detach().float().reshape(c).contiguous()
        self.b_mask = se.conv_mask.bias.detach().float().reshape(1).contiguous()
        self.w1 = se.se_module[0].weight.detach().float().reshape(-1, c).contiguous()
        self.w2 = se.se_module[2].weight.detach().float().reshape(c, -1).contiguous()


class RepVGGPluXNetwork(nn.Module):
    def __init__(self, in_channels_list: List[int], out_channels_list: List[int], groups: int = 4,
                 norm_layer: nn.Module = nn.BatchNorm2d, activation: nn.Module = nn.SiLU, extra_block: bool = False):
        super().__init__()
        for idx in range(len(in_channels_list)):
            if in_channels_list[idx] == 0:
                raise ValueError("in_channels=0 is currently not supported")
        self.lateral_convs = nn.ModuleList()
        self.layer_blocks = nn.ModuleList()
        for idx in range(1, len(out_channels_list)):
            self.lateral_convs.append(Conv2dNormActivation(out_channels_list[idx], out_channels_list[idx - 1], kernel_size=1,
                                                           stride=1, norm_layer=norm_layer, activation_layer=activation,
                                                           inplace=True))
            self.layer_blocks.append(CSPRepPluXLayer(out_channels_list[idx - 1] * 2, out_channels_list[idx - 1], groups=groups,
                                                     norm_layer=norm_layer, activation_layer=activation))
        self.downsample_blocks = nn.ModuleList()
        self.pan_blocks = nn.ModuleList()
        for idx in range(len(in_channels_list) - 1):
            self.downsample_blocks.append(Conv2dNormActivation(out_channels_list[idx], out_channels_list[idx + 1], kernel_size=3,
                                                               stride=2, padding=1, norm_layer=norm_layer,
                                                               activation_layer=activation, inplace=True))
            self.pan_blocks.append(CSPRepPluXLayer(out_channels_list[idx + 1] * 2, out_channels_list[idx + 1], groups=groups,
                                                   norm_layer=norm_layer, activation_layer=activation))
        self.extra_block = extra_block
        self.groups = groups
        self._activation = activation
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight, a=1)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def forward(self, x: OrderedDict):
        keys = list(x.keys())
        x = list(x.values())
        assert len(x) == len(self.layer_blocks) + 1
        # top down path
        results = x
        inner_outs = [results[-1]]
        for idx in range(len(results) - 1, 0, -1):
            feat_high = inner_outs[0]
            feat_low = results[idx - 1]
            feat_high = self.lateral_convs[idx - 1](feat_high)
            inner_outs[0] = feat_high
            upsample_feat = F.interpolate(feat_high, size=feat_low.shape[-2:], mode="nearest")
            inner_out = self.layer_blocks[idx - 1](torch.cat([upsample_feat, feat_low], dim=1))
            inner_outs.insert(0, inner_out)
        # bottom up path
        results = [inner_outs[0]]
        for idx in range(len(inner_outs) - 1):
            feat_low = results[-1]
            feat_high = inner_outs[idx + 1]
            downsample_feat = self.downsample_blocks[idx](feat_low)
            out = self.pan_blocks[idx](torch.cat([downsample_feat, feat_high], dim=1))
            results.append(out)
        output = OrderedDict()
        for idx in range(len(x)):
            output[keys[idx]] = results[idx]
        if self.extra_block:
            output["pool"] = F.max_pool2d(list(output.values())[-1], 1, 2, 0)
        return output

    # ---- token-layout inference and training ---------------------------------------------------------------------------
    def _autograd_records(self, memory: Tensor) -> bool:
        return torch.is_grad_enabled() and (memory.requires_grad or any(p.requires_grad for p in self.parameters()))

    def _tokens_structure_ok(self, memory: Tensor, shapes_list, norms) -> bool:
        """the structural conditions of both token paths; ``norms``: the BatchNorm types accepted"""
        if self.extra_block or not memory.is_cuda or memory.dtype != torch.float32 or memory.dim() != 3:
            return False
        c = memory.shape[2]
        if len(shapes_list) != len(self.layer_blocks) + 1 or len(shapes_list) < 2 or c % self.groups or (c // self.groups) % 64:
            return False
        for m in self.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm) and type(m) not in norms:
                return False
            if isinstance(m, Conv2dNormActivation):
                if m[0].in_channels not in (c, 2 * c) or m[0].out_channels != c or m[0].dilation != (1, 1):
                    return False
                if len(m) < 2 or type(m[1]) not in norms or (len(m) == 3 and type(m[2]) is not nn.SiLU):
                    return False
        for layer in list(self.layer_blocks) + list(self.pan_blocks):
            if not isinstance(layer.conv3, nn.Identity) or len(layer.bottlenecks) == 0:
                return False
            for blk in layer.bottlenecks:
                if not isinstance(blk.identity, nn.Identity) or type(blk.activation) is not nn.SiLU:
                    return False
        for (h, w), (h2, w2) in zip(shapes_list[:-1], shapes_list[1:]):
            if ((h - 1) // 2 + 1, (w - 1) // 2 + 1) != (h2, w2):
                return False
        return True

    def tokens_supported(self, memory: Tensor, shapes_list: Sequence[Tuple[int, int]]) -> bool:
        """True when forward_tokens can run this call on the folded eval weights: eval mode, CUDA fp32 memory, no autograd, no
        extra block, one channel width C at every level with C / groups a multiple of 64, the reference's BatchNorm / SiLU
        layers, CSP layers without conv3 and with at least one block, and stride-2 downsampling that lands on the next level's
        shape (as the reference's concatenation needs)."""
        if self.training or self._autograd_records(memory):
            return False
        return self._tokens_structure_ok(memory, shapes_list, (nn.BatchNorm2d,))

    def training_tokens_supported(self, memory: Tensor, shapes_list: Sequence[Tuple[int, int]]) -> bool:
        """True when forward_tokens runs this call with the reference's op structure under autograd: training mode or autograd
        recording, the structure tokens_supported asks for (BatchNorm2d or SyncBatchNorm layers), fp32 CUDA parameters and
        convolutions without bias."""
        if not (self.training or self._autograd_records(memory)):
            return False
        if any(not p.is_cuda or p.dtype != torch.float32 for p in self.parameters()):
            return False
        if any(isinstance(m, Conv2dNormActivation) and m[0].bias is not None for m in self.modules()):
            return False
        return self._tokens_structure_ok(memory, shapes_list, (nn.BatchNorm2d, nn.SyncBatchNorm))

    def _kernel_weights(self):
        """folded eval weights in kernel form, rebuilt when any parameter or buffer changes (in place or replaced)"""
        def build():
            def conv(wb, groups=1, stride=1):  # (weight, bias) folded in float64
                return TokenConv(wb[0].float(), wb[1].float(), groups, stride, cabi.ACT_SILU)
            f = dict(lateral=[conv(fold_conv_norm(m, torch.float64)) for m in self.lateral_convs],
                     down=[conv(fold_conv_norm(m, torch.float64), stride=2) for m in self.downsample_blocks])
            for name in ("layer_blocks", "pan_blocks"):
                f[name] = [(conv(fold_csp_projection(layer, torch.float64)),
                            [(conv(fold_repvgg(blk, torch.float64), blk.conv1[0].groups), _KGate(blk.se_module))
                             for blk in layer.bottlenecks]) for layer in getattr(self, name)]
            return f
        return derived.cached(self, "kernel_weights", list(self.parameters()) + list(self.buffers()), build)

    @staticmethod
    def launches_per_forward(levels: int = 4, blocks: int = 3) -> int:
        """library launches of one forward_tokens: per convolution 2 (activation scale + convolution), per context gate 3,
        per top-down step one more for the upsample-concat operand (plus one memset of the output)"""
        csp = 2 + blocks * (2 + 3)
        return (levels - 1) * ((2 + 1 + csp) + (2 + csp))

    def _csp(self, f, x: Tensor, hw, dst: Tensor):
        proj_conv, blocks = f
        proj = proj_conv(x, hw, cabi.pow2_scale(x, 12))  # (b, HW, 2C): [SiLU(BN(conv1(x))) | SiLU(BN(conv2(x)))]
        c = proj.shape[2] // 2
        cur, base = proj[:, :, :c], proj
        for i, (conv, gate) in enumerate(blocks):
            y = conv(cur, hw, cabi.pow2_scale(base, 12))
            last = i == len(blocks) - 1
            cur = cabi.context_gate(y, cur, gate.w_mask, gate.b_mask, gate.w1, gate.w2, z=proj[:, :, c:] if last else None,
                                    out=dst if last else None)
            base = cur
        return dst

    def _conv_norm_act_rows(self, m: Conv2dNormActivation, x: Tensor, a_scale: Tensor, hw, stride: int = 1) -> Tensor:
        pad, k = m[0].kernel_size[0] // 2, m[0].kernel_size[0]
        y = _norm_rows(m[1], _TokenConv2d.apply(x, m[0].weight, a_scale, hw, stride),
                       [(v + 2 * pad - k) // stride + 1 for v in hw])
        return m[2](y) if len(m) > 2 else y

    def _csp_rows(self, layer: CSPRepPluXLayer, x: Tensor, hw) -> Tensor:
        x_scale = cabi.pow2_scale(x, 12)
        h = self._conv_norm_act_rows(layer.conv1, x, x_scale, hw)
        for blk in layer.bottlenecks:
            h_scale = cabi.pow2_scale(h, 12)
            y = _norm_rows(blk.conv1[1], _TokenConv2d.apply(h, blk.conv1[0].weight, h_scale, hw, 1), hw)
            y = y + blk.alpha * _norm_rows(blk.conv2[1], _TokenConv2d.apply(h, blk.conv2[0].weight, h_scale, hw, 1), hw)
            h = _gate_rows(blk.se_module, blk.activation(y)) + h
        return h + self._conv_norm_act_rows(layer.conv2, x, x_scale, hw)

    def _forward_tokens_autograd(self, memory: Tensor, shapes_list, lv) -> Tensor:
        """forward()'s op structure on token rows (training_tokens_supported)"""
        levels = len(shapes_list)
        lat = [None] * levels
        feat_high, src = lv[-1], memory
        for idx in range(levels - 1, 0, -1):
            lat[idx] = self._conv_norm_act_rows(self.lateral_convs[idx - 1], feat_high, cabi.pow2_scale(src, 12), shapes_list[idx])
            cat = _UpsampleConcat.apply(lat[idx], shapes_list[idx], lv[idx - 1], shapes_list[idx - 1])
            feat_high = src = self._csp_rows(self.layer_blocks[idx - 1], cat, shapes_list[idx - 1])
        outs = [feat_high]
        for idx in range(levels - 1):
            down = self._conv_norm_act_rows(self.downsample_blocks[idx], outs[-1], cabi.pow2_scale(outs[-1], 12), shapes_list[idx],
                                            stride=2)
            outs.append(self._csp_rows(self.pan_blocks[idx], torch.cat([down, lat[idx + 1]], 2), shapes_list[idx + 1]))
        return torch.cat(outs, 1)

    def forward_tokens(self, memory: Tensor, shapes_list: Sequence[Tuple[int, int]]) -> Tensor:
        """The neck on the encoder memory (b, Nv, C) with levels of shapes_list in token order -> (b, Nv, C), the values of
        forward() on the NCHW maps.  Eval without autograd runs the folded weights (tokens_supported); training or autograd the
        reference's op structure (training_tokens_supported).  No host synchronisation: capturable in a CUDA graph."""
        folded = self.tokens_supported(memory, shapes_list)
        if not folded and not self.training_tokens_supported(memory, shapes_list):
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported / training_tokens_supported)")
        memory = memory.contiguous()
        b, nv, c = memory.shape
        shapes_list = [tuple(int(v) for v in s) for s in shapes_list]
        sizes = [h * w for h, w in shapes_list]
        starts = [sum(sizes[:i]) for i in range(len(sizes))]
        if sum(sizes) != nv:
            raise RuntimeError(f"forward_tokens: memory has {nv} tokens, the levels {sum(sizes)}")
        levels = len(sizes)
        lv = [memory[:, s:s + n] for s, n in zip(starts, sizes)]
        if not folded:
            return self._forward_tokens_autograd(memory, shapes_list, lv)
        f = self._kernel_weights()
        out = torch.zeros_like(memory)  # zero: the activation scale of a level slice is taken over the whole tensor
        outs = [out[:, s:s + n] for s, n in zip(starts, sizes)]
        # bottom-up operands [downsample(previous output) | lateral output] of levels 1..L-1: the lateral convolutions of the
        # top-down path write their half directly
        bu = [None] + [torch.empty(b, n, 2 * c, device=memory.device, dtype=torch.float32) for n in sizes[1:]]
        feat_high, base = lv[-1], memory
        for idx in range(levels - 1, 0, -1):
            lat = bu[idx][:, :, c:]
            f["lateral"][idx - 1](feat_high, shapes_list[idx], cabi.pow2_scale(base, 12), out=lat)
            cat = cabi.upsample_nearest_concat(lat, shapes_list[idx], lv[idx - 1], shapes_list[idx - 1])
            dst = outs[0] if idx == 1 else torch.empty(b, sizes[idx - 1], c, device=memory.device, dtype=torch.float32)
            self._csp(f["layer_blocks"][idx - 1], cat, shapes_list[idx - 1], dst)
            feat_high, base = dst, dst
        for idx in range(levels - 1):
            f["down"][idx](outs[idx], shapes_list[idx], cabi.pow2_scale(out, 12), out=bu[idx + 1][:, :, :c])
            self._csp(f["pan_blocks"][idx], bu[idx + 1], shapes_list[idx + 1], outs[idx + 1])
        return out
