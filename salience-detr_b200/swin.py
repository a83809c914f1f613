"""Swin Transformer backbone (models/backbones/swin.py:SwinTransformerBackbone of the original project), used by the Swin-L
config (configs/salience_detr/salience_detr_swin_l_800_1333.py).

The network classes are torchvision's public Swin Transformer (``SwinTransformer``, ``SwinTransformerBlock``,
``ShiftedWindowAttention``, ``PatchMerging``, their V2 variants and ``torchvision.ops.MLP``), which is what the reference's
module holds.  ``SwinTransformerBackbone(arch, weights, return_indices, freeze_indices, **kwargs)`` is an ``nn.Module`` whose
``features`` are the network's up to the last returned stage (the stem ``features.0``, stage ``i`` at ``features.{2i+1}``, the
PatchMerging after it at ``features.{2i+2}``; no ``norm``, no ``head``), so its ``state_dict`` has exactly the reference feature
extractor's keys and shapes, ``relative_position_index`` buffers included.  The full network is built and initialised as the
reference does it, in the same RNG order, so a seed gives the reference's tensors.  ``forward(x)`` returns
``{"features.{2i+1}": map}`` for ``i`` in ``return_indices``, in that order, each the ``permute(0, 3, 1, 2)`` of a BHWC tensor.

``forward`` is the reference's op chain in torch, ``forward_torch(x)``, whenever ``tokens_supported(x)`` does not hold: with
autograd, on the CPU, with active stochastic depth or dropout, for the V2 archs (post-norm, cosine attention, a CPB MLP), and
for the 96-wide stages of swin_t / swin_s.  Otherwise it is ``forward_tokens(x)``, on token rows ``(b, h*w, C)`` in raster
order:

- the stem (``sdetr_convnext_stem``): conv 4x4 / 4 and its LayerNorm in fp32 FMAs, read straight from the NCHW batch;
- per block 11 launches: norm1 (``sdetr_layernorm_tokens``) and its scale, the QKV Linear, the shifted-window attention
  (``sdetr_window_attention_tokens``: padding, roll, windows, relative position bias and shift mask in index arithmetic) and its
  scale, the output projection with the residual written over the block input, norm2 and its scale, fc1 and its scale, and fc2
  with exact GELU applied as it loads and the residual (every Linear on ``sdetr_gemm_f16x3_ex``, the persistent 3xFP16
  projection GEMM: fp32-class accuracy whatever ``allow_tf32`` says);
- per PatchMerging 3 launches: the padded 2x2 concatenation and its LayerNorm over 4C (``sdetr_patch_merge_layernorm_tokens``),
  its scale, and the reduction GEMM.

Each returned map is a channels-last NCHW view of its own ``(b, h*w, C)`` token buffer, which ``ChannelMapper`` reads in place.
The derived weights (every Linear's fp16 pair, each block's relative position bias expanded to (nH, N, N)) are cached per
parameter version through ``derived.cached``.  No host synchronisation: the call can be captured in a CUDA graph.
"""
from __future__ import annotations

import inspect
from typing import Tuple

from torch import Tensor, nn
from torchvision.models.swin_transformer import (  # noqa: F401  (the reference module's classes)
    PatchMerging,
    PatchMergingV2,
    ShiftedWindowAttention,
    ShiftedWindowAttentionV2,
    SwinTransformer,
    SwinTransformerBlock,
    SwinTransformerBlockV2,
    shifted_window_attention,
)
from torchvision.ops import MLP, Permute

from . import cabi
from .token_backbone import FeatureBackbone, tokens_ready


class _KBlock:
    """one SwinTransformerBlock in kernel form: both LayerNorms, the four Linears as fp16 pairs with device scales and their
    biases, and the relative position bias expanded to (nH, N, N) from the block's own index buffer"""

    def __init__(self, blk: SwinTransformerBlock):
        attn, fc1, fc2 = blk.attn, blk.mlp[0], blk.mlp[3]
        self.ln1 = (blk.norm1.weight.detach(), blk.norm1.bias.detach(), blk.norm1.eps)
        self.ln2 = (blk.norm2.weight.detach(), blk.norm2.bias.detach(), blk.norm2.eps)
        self.wqkv, self.bqkv = cabi.split_f16_pair_dev(attn.qkv.weight.detach()), attn.qkv.bias.detach()
        self.wproj, self.bproj = cabi.split_f16_pair_dev(attn.proj.weight.detach()), attn.proj.bias.detach()
        self.w1, self.b1 = cabi.split_f16_pair_dev(fc1.weight.detach()), fc1.bias.detach()
        self.w2, self.b2 = cabi.split_f16_pair_dev(fc2.weight.detach()), fc2.bias.detach()
        self.heads, self.window, self.shift = attn.num_heads, tuple(attn.window_size), tuple(attn.shift_size)
        n = self.window[0] * self.window[1]
        table = attn.relative_position_bias_table.detach()
        self.rel_bias = table[attn.relative_position_index].view(n, n, -1).permute(2, 0, 1).contiguous()


class _KMerge:
    """one PatchMerging in kernel form: its LayerNorm over 4C and the reduction weight as an fp16 pair"""

    def __init__(self, pm: PatchMerging):
        self.ln = (pm.norm.weight.detach(), pm.norm.bias.detach(), pm.norm.eps)
        self.w = cabi.split_f16_pair_dev(pm.reduction.weight.detach())


class SwinTransformerBackbone(FeatureBackbone):
    # name -> SwinTransformer arguments (the reference's model_arch table, without the download URLs)
    model_arch = {
        "swin_t": dict(patch_size=(4, 4), embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=(7, 7),
                       stochastic_depth_prob=0.2),
        "swin_s": dict(patch_size=(4, 4), embed_dim=96, depths=(2, 2, 18, 2), num_heads=(3, 6, 12, 24), window_size=(7, 7),
                       stochastic_depth_prob=0.3),
        "swin_b": dict(patch_size=(4, 4), embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=(7, 7),
                       stochastic_depth_prob=0.5),
        "swin_l": dict(patch_size=(4, 4), embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window_size=(7, 7),
                       stochastic_depth_prob=0.2),
        "swin_b_384": dict(patch_size=(4, 4), embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32),
                           window_size=(12, 12), stochastic_depth_prob=0.2),
        "swin_l_384": dict(patch_size=(4, 4), embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48),
                           window_size=(12, 12), stochastic_depth_prob=0.2),
        "swin_v2_t": dict(patch_size=[4, 4], embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=[8, 8],
                          stochastic_depth_prob=0.2, block=SwinTransformerBlockV2, downsample_layer=PatchMergingV2),
        "swin_v2_b": dict(patch_size=[4, 4], embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=[8, 8],
                          stochastic_depth_prob=0.5, block=SwinTransformerBlockV2, downsample_layer=PatchMergingV2),
    }
    network, skip_prefixes, kblock, kdown = SwinTransformer, ("norm.", "head."), _KBlock, _KMerge

    def _config(self, arch: str, kwargs: dict) -> dict:
        # as the reference merges them: a keyword argument of SwinTransformer overrides the arch's value unless it is None
        names = inspect.signature(SwinTransformer).parameters
        unknown = [k for k in kwargs if k not in names]
        if unknown:
            raise TypeError(f"SwinTransformerBackbone: unexpected keyword arguments {unknown}")
        return {**self.model_arch[arch], **{k: v for k, v in kwargs.items() if v is not None}}

    @staticmethod
    def _stage_channels(cfg: dict, i: int) -> int:
        return cfg["embed_dim"] * 2 ** i

    @staticmethod
    def _nchw(x: Tensor) -> Tensor:
        return x.permute(0, 3, 1, 2)

    # ---- token-layout inference --------------------------------------------------------------------------------------
    def tokens_supported(self, x) -> bool:
        """True when forward_tokens can run this call: a CUDA fp32 NCHW-contiguous (b, 3, H, W) input whose every map is at least
        1x1, parameters fp32 on its device, nothing that needs a gradient (autograd off, or neither the input nor a parameter
        requires one), no active stochastic depth, dropout or attention dropout (train mode with p > 0), and
        layers_supported()."""
        if not tokens_ready(self, x) or x.shape[2] < 4 or x.shape[3] < 4:
            return False
        for m in self.features.modules():
            if isinstance(m, SwinTransformerBlock):
                if m.stochastic_depth.training and m.stochastic_depth.p > 0:
                    return False
                if m.attn.training and (m.attn.dropout > 0 or m.attn.attention_dropout > 0):
                    return False
            elif isinstance(m, nn.Dropout) and m.training and m.p > 0:
                return False
        return self.layers_supported()

    def layers_supported(self) -> bool:
        """The layer half of tokens_supported: the default stem, V1 blocks and PatchMerging (nn.LayerNorm with affine weights,
        exact GELU), head dim 32, windows of at most 144 tokens with shifts inside them, and stage widths that are multiples of
        64 up to 1536."""
        def ln_ok(n, c):
            return type(n) is nn.LayerNorm and n.normalized_shape == (c,) and n.weight is not None and n.bias is not None

        def width_ok(c):
            return c % 64 == 0 and 0 < c <= 1536

        def linear_ok(lin, cin, cout, bias=True):
            return type(lin) is nn.Linear and (lin.in_features, lin.out_features) == (cin, cout) and (lin.bias is not None) == bias

        stem = self.features[0]
        if not (type(stem) is nn.Sequential and len(stem) == 3 and type(stem[0]) is nn.Conv2d and type(stem[1]) is Permute):
            return False
        conv = stem[0]
        c = conv.out_channels
        if (conv.kernel_size, conv.stride, conv.padding, conv.dilation, conv.groups) != ((4, 4), (4, 4), (0, 0), (1, 1), 1):
            return False
        if conv.in_channels != 3 or conv.bias is None or list(stem[1].dims) != [0, 2, 3, 1] or not width_ok(c) or not ln_ok(stem[2], c):
            return False
        for i in range(self._num_stages()):
            for blk in self.features[2 * i + 1]:
                if type(blk) is not SwinTransformerBlock or type(blk.attn) is not ShiftedWindowAttention:
                    return False
                attn, mlp = blk.attn, blk.mlp
                if not (ln_ok(blk.norm1, c) and ln_ok(blk.norm2, c) and attn.num_heads * 32 == c):
                    return False
                if not (linear_ok(attn.qkv, c, 3 * c) and linear_ok(attn.proj, c, c)):
                    return False
                win, shift = list(attn.window_size), list(attn.shift_size)
                if len(win) != 2 or len(shift) != 2 or not all(0 < w and 0 <= s < w for w, s in zip(win, shift)):
                    return False
                n = win[0] * win[1]
                if n > 144 or tuple(attn.relative_position_index.shape) != (n * n,):
                    return False
                if attn.relative_position_bias_table.dim() != 2 or attn.relative_position_bias_table.shape[1] != attn.num_heads:
                    return False
                if not (type(mlp) is MLP and len(mlp) == 5 and type(mlp[1]) is nn.GELU and mlp[1].approximate == "none"):
                    return False
                hidden = mlp[0].out_features
                if hidden % 64 != 0 or not (linear_ok(mlp[0], c, hidden) and linear_ok(mlp[3], hidden, c)):
                    return False
            if i + 1 < self._num_stages():
                pm = self.features[2 * i + 2]
                if type(pm) is not PatchMerging or not ln_ok(pm.norm, 4 * c) or not linear_ok(pm.reduction, 4 * c, 2 * c, False):
                    return False
                if not width_ok(2 * c):
                    return False
                c = 2 * c
        return True

    def launches_per_forward(self) -> int:
        """library launches of one forward_tokens: the stem, 11 per block (norm1, scale, QKV, window attention, scale, proj,
        norm2, scale, fc1, scale, fc2) and 3 per PatchMerging between kept stages (merge LayerNorm, scale, reduction)"""
        n = 1
        for i in range(self._num_stages()):
            n += 11 * len(self.features[2 * i + 1]) + (3 if i + 1 < self._num_stages() else 0)
        return n

    @staticmethod
    def _block_tokens(k: _KBlock, t: Tensor, hw: Tuple[int, int]) -> Tensor:
        # t = t + proj(attention(norm1(t))), then t = t + fc2(GELU(fc1(norm2(t)))): written over the block input
        u = cabi.layernorm_tokens(t, *k.ln1)
        qkv = cabi.gemm_f16x3_ex(u, cabi.pow2_scale(u, 12), *k.wqkv, k.bqkv)
        a = cabi.window_attention_tokens(qkv, hw, k.bqkv, k.rel_bias, k.heads, k.window, k.shift)
        cabi.gemm_f16x3_ex(a, cabi.pow2_scale(a, 12), *k.wproj, k.bproj, z=t, out=t)
        u = cabi.layernorm_tokens(t, *k.ln2)
        h = cabi.gemm_f16x3_ex(u, cabi.pow2_scale(u, 12), *k.w1, k.b1)
        return cabi.gemm_f16x3_ex(h, cabi.pow2_scale(h, 12), *k.w2, k.b2, act=cabi.ACT_GELU, z=t, out=t)

    @staticmethod
    def _down_tokens(pm: _KMerge, t: Tensor, hw: Tuple[int, int]) -> Tensor:
        r = cabi.patch_merge_layernorm_tokens(t, hw, *pm.ln)
        return cabi.gemm_f16x3_ex(r, cabi.pow2_scale(r, 12), *pm.w)

    @staticmethod
    def _down_hw(hw: Tuple[int, int]) -> Tuple[int, int]:
        return (hw[0] + 1) // 2, (hw[1] + 1) // 2
