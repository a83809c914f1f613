"""FocalNet backbone (models/backbones/focalnet.py:FocalNetBackbone of the original project), used by the FocalNet-L config
(configs/salience_detr/salience_detr_focalnet_large_lrf_800_1333.py).

The network follows the public Focal Modulation Networks (``FocalNet``, ``PatchEmbed``, ``FocalModulationBlock``,
``FocalModulation``, ``Mlp``), with the reference's attribute names and construction order, so a seed gives the reference's
tensors.  ``FocalNetBackbone(arch, weights, return_indices, freeze_indices, **kwargs)`` is, like the reference's, an
``nn.Sequential`` of the feature extractor ``0`` (the network's ``patch_embed`` and ``layers`` up to the last returned stage,
without that stage's ``downsample``) and ``1``, the post-process LayerNorms ``norm{i}`` of the returned stages, so its
``state_dict`` has exactly the reference's keys and shapes.  ``forward(x)`` returns ``{"layers.{i}.blocks": map}`` for ``i`` in
``return_indices``, in that order, each ``norm{i}`` of the stage output as an NCHW map.

``forward`` is the reference's op chain in torch, ``forward_torch(x)``, whenever ``tokens_supported(x)`` does not hold: with
autograd, on the CPU, with active stochastic depth or dropout, and for every arch but ``focalnet_large_lrf`` and
``focalnet_large_lrf_fl4``: tiny, small and base are pre-LN with 4x4 / 2x2 patch convolutions, xlarge reaches width 2048 and
huge has a LayerNorm inside the modulation and width 352.  Otherwise it is ``forward_tokens(x)``, on token rows ``(b, h*w, C)``
in raster order:

- the stem (``sdetr_focalnet_stem``): conv 7x7 / 4, padding 2 on the image padded to a multiple of 4 (a ceil(H / 4) x
  ceil(W / 4) map) and its LayerNorm in fp32 FMAs, read straight from the NCHW batch;
- per block 14 + L launches (L focal levels): ``f`` and its scale, into ``[q | ctx | gates]`` padded with zero rows to 2C + 8
  columns; one ``sdetr_focal_level_tokens`` per level (GELU of the depthwise k x k convolution, ``ctx_all += ctx * gate``, the
  last level's channel sums); ``sdetr_focal_global_context`` (``+ GELU(mean) * gate_L``, ``/ (L + 1)``); ``h`` and its scale;
  ``sdetr_focal_modulate`` (``q * h``); ``proj`` and its scale; ``sdetr_layernorm_scale_add_tokens`` (``t += gamma_1 *
  norm1(.)``); ``fc1`` and its scale; ``fc2`` with exact GELU applied as it loads, and its scale; ``t += gamma_2 * norm2(.)``.
  Every Linear runs on ``sdetr_gemm_f16x3_ex``, the persistent 3xFP16 projection GEMM (fp32-class accuracy whatever
  ``allow_tf32`` says);
- per downsample 3 launches: the scale, the 3x3 / stride-2 convolution (``sdetr_conv2d_f16x3``; the reference's pad to an even
  size adds only zeros it never reads) and its LayerNorm (``sdetr_layernorm_tokens``);
- one ``sdetr_layernorm_tokens`` per returned stage, into a buffer of its own: the un-normalised stage output goes on.

Each returned map is a channels-last NCHW view of its own ``(b, h*w, C)`` token buffer, which ``ChannelMapper`` reads in place.
The derived weights are cached per parameter version through ``derived.cached``.  No host synchronisation: the call can be
captured in a CUDA graph.
"""
from __future__ import annotations

import inspect
from collections import OrderedDict
from functools import partial
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor, nn
from torch.nn.init import trunc_normal_
from torchvision.ops import StochasticDepth

from . import cabi, derived
from .token_backbone import freeze, load_weights, token_maps, tokens_ready


class Mlp(nn.Module):
    """fc1, activation, dropout, fc2, dropout"""

    def __init__(self, in_features, hidden_features=None, out_features=None, activation_layer=nn.GELU, drop=0.0):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = activation_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        return self.drop(self.fc2(self.drop(self.act(self.fc1(x)))))


class FocalModulation(nn.Module):
    """Focal modulation of a (B, H, W, C) map: ``f`` projects to the query, the context and L + 1 gates; level l runs a depthwise
    (focal_factor l + focal_window)-wide convolution and GELU on the context and adds it, gated, to ctx_all; the gated GELU of
    the last level's global mean is added last.  ``h`` (a 1x1 convolution) of ctx_all modulates the query, and ``proj`` maps back."""

    def __init__(self, dim: int, proj_drop=0.0, focal_level=2, focal_window=7, focal_factor=2, use_postln_in_modulation=False,
                 normalize_modulator=False):
        super().__init__()
        self.dim = dim
        self.focal_level = focal_level
        self.focal_window = focal_window
        self.focal_factor = focal_factor
        self.use_postln_in_modulation = use_postln_in_modulation
        self.normalize_modulator = normalize_modulator
        self.f = nn.Linear(dim, 2 * dim + focal_level + 1)
        self.h = nn.Conv2d(dim, dim, kernel_size=1, stride=1, padding=0, groups=1)
        self.act = nn.GELU()
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)
        self.focal_layers = nn.ModuleList()
        if use_postln_in_modulation:
            self.ln = nn.LayerNorm(dim)
        for k in range(focal_level):
            ks = focal_factor * k + focal_window
            self.focal_layers.append(nn.Sequential(
                nn.Conv2d(dim, dim, kernel_size=ks, stride=1, groups=dim, padding=ks // 2, bias=False), nn.GELU()))

    def forward(self, x):
        C = x.shape[-1]
        x = self.f(x).permute(0, 3, 1, 2).contiguous()
        q, ctx, gates = torch.split(x, (C, C, self.focal_level + 1), 1)
        ctx_all = 0
        for level in range(self.focal_level):
            ctx = self.focal_layers[level](ctx)
            ctx_all = ctx_all + ctx * gates[:, level:level + 1]
        ctx_global = self.act(ctx.mean(2, keepdim=True).mean(3, keepdim=True))
        ctx_all = ctx_all + ctx_global * gates[:, self.focal_level:]
        if self.normalize_modulator:
            ctx_all = ctx_all / (self.focal_level + 1)
        x_out = (q * self.h(ctx_all)).permute(0, 2, 3, 1).contiguous()
        if self.use_postln_in_modulation:
            x_out = self.ln(x_out)
        return self.proj_drop(self.proj(x_out))


class FocalModulationBlock(nn.Module):
    """Post-LN (use_postln): x + gamma_1 * norm1(modulation(x)), then x + gamma_2 * norm2(mlp(x)); pre-LN: the norms before
    the branches.  Stochastic depth on both branches; gamma_1 / gamma_2 learnable (init 1e-4) with use_layerscale, else 1."""

    def __init__(self, dim: int, mlp_ratio: float = 4.0, focal_level: int = 2, focal_window: int = 9, dropout: float = 0.0,
                 stochastic_depth_prob: float = 0.0, norm_layer=nn.LayerNorm, use_postln: bool = False,
                 use_postln_in_modulation: bool = False, normalize_modulator: bool = False, use_layerscale: bool = False):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.modulation = FocalModulation(dim, focal_window=focal_window, focal_level=focal_level, proj_drop=dropout,
                                          use_postln_in_modulation=use_postln_in_modulation,
                                          normalize_modulator=normalize_modulator)
        self.drop_path = StochasticDepth(stochastic_depth_prob, "row")
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), activation_layer=nn.GELU, drop=dropout)
        if use_layerscale:
            self.gamma_1 = nn.Parameter(torch.full((dim,), 1e-4))
            self.gamma_2 = nn.Parameter(torch.full((dim,), 1e-4))
        else:
            self.gamma_1 = self.gamma_2 = 1.0
        self.use_postln = use_postln

    def forward(self, x):
        if self.use_postln:
            x = x + self.drop_path(self.gamma_1 * self.norm1(self.modulation(x)))
            return x + self.drop_path(self.gamma_2 * self.norm2(self.mlp(x)))
        x = x + self.drop_path(self.gamma_1 * self.modulation(self.norm1(x)))
        return x + self.drop_path(self.gamma_2 * self.mlp(self.norm2(x)))


class PatchEmbed(nn.Module):
    """(N, H, W, C) -> zero-pad right and bottom to a multiple of patch_size, convolution, LayerNorm -> (N, H', W', C').  With
    use_conv_embed the convolution is 7x7 / 4, padding 2 for the stem and 3x3 / 2, padding 1 otherwise; else patch_size-wide
    patches."""

    def __init__(self, in_channels: int, hidden_channels: int, patch_size=(4, 4), norm_layer=nn.LayerNorm,
                 use_conv_embed: bool = False, is_stem: bool = False):
        super().__init__()
        self.patch_size = patch_size
        if use_conv_embed and is_stem:
            self.proj = nn.Conv2d(in_channels, hidden_channels, kernel_size=7, stride=4, padding=2)
        elif use_conv_embed:
            self.proj = nn.Conv2d(in_channels, hidden_channels, kernel_size=3, stride=2, padding=1)
        else:
            self.proj = nn.Conv2d(in_channels, hidden_channels, kernel_size=patch_size, stride=patch_size)
        self.norm = norm_layer(hidden_channels)

    def forward(self, x):
        H, W = x.shape[-3], x.shape[-2]
        pad_r = (self.patch_size[1] - W % self.patch_size[1]) % self.patch_size[1]
        pad_b = (self.patch_size[0] - H % self.patch_size[0]) % self.patch_size[0]
        x = F.pad(x, (0, 0, 0, pad_r, 0, pad_b))
        x = self.proj(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        return self.norm(x)


class FocalNet(nn.Module):
    """Focal Modulation Networks (arXiv:2203.11926) without the classifier: ``patch_embed``, ``pos_drop`` and ``layers``, stage i
    an ``nn.Sequential`` of ``blocks`` (embed_dim 2^i wide) and, but for the last stage, the ``downsample`` PatchEmbed to twice
    the width.  Linears trunc_normal_(std 0.02) with zero biases, LayerNorms (1, 0), convolutions torch's default."""

    def __init__(self, patch_size: List[int], embed_dim: int, depths: List[int], mlp_ratio: float = 4.0, dropout: float = 0.0,
                 stochastic_depth_prob: float = 0.3, norm_layer=partial(nn.LayerNorm, eps=1e-5), focal_levels=(3, 3, 3, 3),
                 focal_windows=(3, 3, 3, 3), use_conv_embed=False, use_postln=False, use_postln_in_modulation=False,
                 use_layerscale=False, normalize_modulator=False):
        super().__init__()
        self.num_layers = len(depths)
        self.patch_embed = PatchEmbed(3, embed_dim, patch_size, norm_layer, use_conv_embed, is_stem=True)
        self.pos_drop = nn.Dropout(p=dropout)
        self.layers = nn.ModuleList()
        total = sum(depths)
        block_id = 0
        for i in range(len(depths)):
            dim = embed_dim * 2 ** i
            blocks = []
            for _ in range(depths[i]):
                blocks.append(FocalModulationBlock(
                    dim, mlp_ratio=mlp_ratio, focal_level=focal_levels[i], focal_window=focal_windows[i], dropout=dropout,
                    stochastic_depth_prob=stochastic_depth_prob * float(block_id) / (total - 1), norm_layer=norm_layer,
                    use_postln=use_postln, use_postln_in_modulation=use_postln_in_modulation,
                    normalize_modulator=normalize_modulator, use_layerscale=use_layerscale))
                block_id += 1
            stage = OrderedDict(blocks=nn.Sequential(*blocks))
            if i < len(depths) - 1:
                stage["downsample"] = PatchEmbed(dim, 2 * dim, (2, 2), norm_layer, use_conv_embed)
            self.layers.append(nn.Sequential(stage))
        self.apply(self._init_weights)

    def forward(self, x):
        """(b, 3, H, W) -> the last stage's (b, h, w, C) map"""
        x = self.pos_drop(self.patch_embed(x.permute(0, 2, 3, 1)))
        for i in range(self.num_layers):
            x = self.layers[i](x)
        return x

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)


class PostProcess(nn.Module):
    """one LayerNorm ``norm{i}`` per returned stage i"""

    def __init__(self, in_channels, return_indices=(0, 1, 2, 3), norm_layer=nn.LayerNorm):
        super().__init__()
        self.return_indices = return_indices
        for channel, idx in zip(in_channels, return_indices):
            self.add_module(f"norm{idx}", norm_layer(channel))


def _ln_ok(n, c):
    return type(n) is nn.LayerNorm and n.normalized_shape == (c,) and n.weight is not None and n.bias is not None


def _linear_ok(lin, cin, cout):
    return type(lin) is nn.Linear and (lin.in_features, lin.out_features) == (cin, cout) and lin.bias is not None


def _conv_ok(conv, cin, cout, k, s, p, groups=1, bias=True):
    return (type(conv) is nn.Conv2d and (conv.in_channels, conv.out_channels, conv.groups) == (cin, cout, groups)
            and conv.kernel_size == (k, k) and conv.stride == (s, s) and conv.padding == (p, p) and conv.dilation == (1, 1)
            and conv.padding_mode == "zeros" and (conv.bias is not None) == bias)


def _gelu_ok(m):
    return type(m) is nn.GELU and m.approximate == "none"


class _KBlock:
    """one post-LN FocalModulationBlock in kernel form: f padded with zero rows to 2C + 8 outputs (q, ctx and the gates on
    16-byte boundaries), the focal levels' depthwise weights as (k * k, C), h, proj, fc1 and fc2 as fp16 pairs with device
    scales and their biases, both LayerNorms and both layer scales"""

    def __init__(self, blk: FocalModulationBlock):
        mod = blk.modulation
        c = mod.dim
        self.C, self.levels, self.normalize = c, mod.focal_level, bool(mod.normalize_modulator)
        fw, fb = mod.f.weight.detach(), mod.f.bias.detach()
        self.wf = cabi.split_f16_pair_dev(torch.cat([fw, fw.new_zeros(8 - mod.focal_level - 1, c)]))
        self.bf = torch.cat([fb, fb.new_zeros(8 - mod.focal_level - 1)])
        self.dw = [fl[0].weight.detach().reshape(c, -1).t().contiguous() for fl in mod.focal_layers]
        self.wh, self.bh = cabi.split_f16_pair_dev(mod.h.weight.detach().reshape(c, c)), mod.h.bias.detach()
        self.wproj, self.bproj = cabi.split_f16_pair_dev(mod.proj.weight.detach()), mod.proj.bias.detach()
        self.w1, self.b1 = cabi.split_f16_pair_dev(blk.mlp.fc1.weight.detach()), blk.mlp.fc1.bias.detach()
        self.w2, self.b2 = cabi.split_f16_pair_dev(blk.mlp.fc2.weight.detach()), blk.mlp.fc2.bias.detach()
        self.ln1 = (blk.norm1.weight.detach(), blk.norm1.bias.detach(), blk.norm1.eps)
        self.ln2 = (blk.norm2.weight.detach(), blk.norm2.bias.detach(), blk.norm2.eps)
        self.g1, self.g2 = blk.gamma_1.detach(), blk.gamma_2.detach()


class _KDown:
    """one downsample PatchEmbed in kernel form: the 3x3 weight as the (Cout, 3, 3, Cin) fp16 pair of conv2d_f16x3, its bias and
    its LayerNorm"""

    def __init__(self, pe: PatchEmbed):
        f_hi, f_lo, _, _, scale = cabi.conv2d_f16x3_split_weight(pe.proj.weight.detach(), 1, dgrad=False)
        self.w, self.b = (f_hi, f_lo, scale), pe.proj.bias.detach()
        self.ln = (pe.norm.weight.detach(), pe.norm.bias.detach(), pe.norm.eps)


class FocalNetBackbone(nn.Sequential):
    # name -> FocalNet arguments (the reference's model_arch table, without the download URLs)
    model_arch = {
        "focalnet_tiny_srf": dict(embed_dim=96, patch_size=(4, 4), depths=(2, 2, 6, 2), stochastic_depth_prob=0.2,
                                  focal_levels=(2, 2, 2, 2), focal_windows=(3, 3, 3, 3)),
        "focalnet_tiny_lrf": dict(embed_dim=96, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.2,
                                  focal_levels=(3, 3, 3, 3), focal_windows=(3, 3, 3, 3)),
        "focalnet_small_srf": dict(embed_dim=96, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.3,
                                   focal_levels=(2, 2, 2, 2), focal_windows=(3, 3, 3, 3)),
        "focalnet_small_lrf": dict(embed_dim=96, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.3,
                                   focal_levels=(3, 3, 3, 3), focal_windows=(3, 3, 3, 3)),
        "focalnet_base_srf": dict(embed_dim=128, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                  focal_levels=(2, 2, 2, 2), focal_windows=(3, 3, 3, 3)),
        "focalnet_base_lrf": dict(embed_dim=128, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                  focal_levels=(3, 3, 3, 3), focal_windows=(3, 3, 3, 3)),
        "focalnet_large_lrf": dict(embed_dim=192, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                   focal_levels=(3, 3, 3, 3), focal_windows=(5, 5, 5, 5), use_conv_embed=True, use_postln=True,
                                   use_postln_in_modulation=False, use_layerscale=True, normalize_modulator=False),
        "focalnet_large_lrf_fl4": dict(embed_dim=192, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                       focal_levels=(4, 4, 4, 4), focal_windows=(3, 3, 3, 3), use_conv_embed=True,
                                       use_postln=True, use_postln_in_modulation=False, use_layerscale=True,
                                       normalize_modulator=True),
        "focalnet_xlarge_lrf": dict(embed_dim=256, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                    focal_levels=(3, 3, 3, 3), focal_windows=(5, 5, 5, 5), use_conv_embed=True, use_postln=True,
                                    use_postln_in_modulation=False, use_layerscale=True, normalize_modulator=False),
        "focalnet_xlarge_lrf_fl4": dict(embed_dim=256, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                        focal_levels=(4, 4, 4, 4), focal_windows=(3, 3, 3, 3), use_conv_embed=True,
                                        use_postln=True, use_postln_in_modulation=False, use_layerscale=True,
                                        normalize_modulator=True),
        "focalnet_huge_fl3": dict(embed_dim=352, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                  focal_levels=(3, 3, 3, 3), focal_windows=(3, 3, 3, 3), use_conv_embed=True, use_postln=True,
                                  use_layerscale=True, use_postln_in_modulation=True, normalize_modulator=False),
        "focalnet_huge_fl4": dict(embed_dim=352, patch_size=(4, 4), depths=(2, 2, 18, 2), stochastic_depth_prob=0.5,
                                  focal_levels=(4, 4, 4, 4), focal_windows=(3, 3, 3, 3), use_conv_embed=True, use_postln=True,
                                  use_postln_in_modulation=True, use_layerscale=True, normalize_modulator=False),
    }

    def __init__(self, arch: str, weights=None, return_indices: Tuple[int, ...] = (0, 1, 2, 3), freeze_indices: Tuple = (),
                 **kwargs):
        if arch not in self.model_arch:
            raise ValueError(f"Expected architecture in {list(self.model_arch)} but got {arch}")
        cfg = self._config(arch, kwargs)
        net = FocalNet(**cfg)
        load_weights(net, weights, ("norm.", "head."), type(self).__name__)
        if len(freeze_indices) > 0:
            freeze([net.patch_embed] + [net.layers[i] for i in freeze_indices])
        return_indices = tuple(int(i) for i in return_indices)
        # what the reference's feature extractor keeps: the stages up to the last returned one, without its downsample
        last = max(return_indices)
        net.layers = nn.ModuleList(list(net.layers)[:last + 1])
        if hasattr(net.layers[last], "downsample"):
            del net.layers[last].downsample
        net.num_layers = last + 1
        num_channels = [cfg["embed_dim"] * 2 ** i for i in return_indices]
        super().__init__(net, PostProcess(num_channels, return_indices, cfg["norm_layer"]))
        self.return_indices, self.num_channels = return_indices, num_channels

    @staticmethod
    def _config(arch: str, kwargs: dict) -> dict:
        # as the reference merges them: every FocalNet argument takes the keyword's value unless it is None, else the arch's
        # unless that is None, else FocalNet's default
        names = inspect.signature(FocalNet).parameters
        unknown = [k for k in kwargs if k not in names]
        if unknown:
            raise TypeError(f"FocalNetBackbone: unexpected keyword arguments {unknown}")
        cfg = {}
        for name, p in names.items():
            value = p.default if p.default is not inspect.Parameter.empty else None
            if FocalNetBackbone.model_arch[arch].get(name) is not None:
                value = FocalNetBackbone.model_arch[arch][name]
            if kwargs.get(name) is not None:
                value = kwargs[name]
            cfg[name] = value
        return cfg

    def _num_stages(self) -> int:
        return max(self.return_indices) + 1

    def forward(self, x: Tensor) -> Dict[str, Tensor]:
        if self.tokens_supported(x):
            return self.forward_tokens(x)
        return self.forward_torch(x)

    def forward_torch(self, x: Tensor) -> Dict[str, Tensor]:
        """the reference's op chain in torch: {"layers.{i}.blocks": map} for i in return_indices, NCHW contiguous"""
        net, post = self[0], self[1]
        x = net.pos_drop(net.patch_embed(x.permute(0, 2, 3, 1)))
        feats = {}
        for i in range(self._num_stages()):
            x = net.layers[i].blocks(x)
            feats[i] = x
            if i + 1 < self._num_stages():
                x = net.layers[i].downsample(x)
        return {f"layers.{i}.blocks": getattr(post, f"norm{i}")(feats[i]).permute(0, 3, 1, 2).contiguous()
                for i in self.return_indices}

    # ---- token-layout inference --------------------------------------------------------------------------------------
    def tokens_supported(self, x) -> bool:
        """True when forward_tokens can run this call: a CUDA fp32 NCHW-contiguous (b, 3, H, W) input, parameters fp32 on its
        device, nothing that needs a gradient (autograd off, or neither the input nor a parameter requires one), no active
        stochastic depth or dropout (train mode with p > 0), and layers_supported()."""
        if not tokens_ready(self, x):
            return False
        for m in self.modules():
            if isinstance(m, StochasticDepth) and m.training and m.p > 0:
                return False
            if isinstance(m, nn.Dropout) and m.training and m.p > 0:
                return False
        return self.layers_supported()

    def layers_supported(self) -> bool:
        """The layer half of tokens_supported: the conv stem (7x7 / 4, padding 2) and conv downsamples (3x3 / 2, padding 1) with
        their LayerNorms, post-LN FocalModulationBlocks with layer scales, no LayerNorm inside the modulation, focal kernels of
        3, 5, 7 or 9 with at most 7 levels, exact GELUs, MLP hidden widths that are multiples of 64, and stage widths that are
        multiples of 64 up to 1536: the focalnet_large_lrf and focalnet_large_lrf_fl4 archs."""
        net, post = self[0], self[1]

        def width_ok(c):
            return c % 64 == 0 and 0 < c <= 1536

        pe = net.patch_embed
        c = pe.proj.out_channels
        if not (type(pe) is PatchEmbed and _conv_ok(pe.proj, 3, c, 7, 4, 2) and tuple(pe.patch_size) == (4, 4)
                and width_ok(c) and _ln_ok(pe.norm, c)):
            return False
        for i in range(self._num_stages()):
            for blk in net.layers[i].blocks:
                if type(blk) is not FocalModulationBlock or not blk.use_postln:
                    return False
                if not (isinstance(blk.gamma_1, nn.Parameter) and isinstance(blk.gamma_2, nn.Parameter)
                        and tuple(blk.gamma_1.shape) == (c,) and tuple(blk.gamma_2.shape) == (c,)):
                    return False
                if not (_ln_ok(blk.norm1, c) and _ln_ok(blk.norm2, c)):
                    return False
                mod = blk.modulation
                if type(mod) is not FocalModulation or mod.use_postln_in_modulation or mod.dim != c:
                    return False
                L = mod.focal_level
                if not (1 <= L <= 7 and len(mod.focal_layers) == L and _gelu_ok(mod.act)):
                    return False
                if not (_linear_ok(mod.f, c, 2 * c + L + 1) and _conv_ok(mod.h, c, c, 1, 1, 0) and _linear_ok(mod.proj, c, c)):
                    return False
                for fl in mod.focal_layers:
                    if not (type(fl) is nn.Sequential and len(fl) == 2 and _gelu_ok(fl[1])):
                        return False
                    k = fl[0].kernel_size[0]
                    if k not in (3, 5, 7, 9) or not _conv_ok(fl[0], c, c, k, 1, k // 2, groups=c, bias=False):
                        return False
                mlp = blk.mlp
                hidden = mlp.fc1.out_features
                if not (type(mlp) is Mlp and _gelu_ok(mlp.act) and hidden % 64 == 0 and _linear_ok(mlp.fc1, c, hidden)
                        and _linear_ok(mlp.fc2, hidden, c)):
                    return False
            if i in self.return_indices and not _ln_ok(getattr(post, f"norm{i}", None), c):
                return False
            if i + 1 < self._num_stages():
                ds = net.layers[i].downsample
                if not (type(ds) is PatchEmbed and _conv_ok(ds.proj, c, 2 * c, 3, 2, 1) and width_ok(2 * c)
                        and _ln_ok(ds.norm, 2 * c)):
                    return False
                c = 2 * c
        return True

    def launches_per_forward(self) -> int:
        """library launches of one forward_tokens: the stem, 14 + L per block of L focal levels (f and its scale, the L levels,
        the global context, h and its scale, the modulation, proj and its scale, the norm1 residual, fc1 and its scale, fc2 and
        its scale, the norm2 residual), 3 per downsample between kept stages (scale, convolution, LayerNorm) and one output
        LayerNorm per returned stage"""
        net = self[0]
        n = 1 + len(self.return_indices)
        for i in range(self._num_stages()):
            n += sum(14 + blk.modulation.focal_level for blk in net.layers[i].blocks)
            n += 3 if i + 1 < self._num_stages() else 0
        return n

    def _kernel_weights(self):
        """the stem ((147, C) weight, bias, LayerNorm), per kept stage its blocks and the downsample after it (None after the
        last), and per returned stage its output LayerNorm, rebuilt when any parameter changes"""
        def build():
            net, post = self[0], self[1]
            conv, ln = net.patch_embed.proj, net.patch_embed.norm
            c = conv.out_channels
            stem = (conv.weight.detach().reshape(c, 147).t().contiguous(), conv.bias.detach(), ln.weight.detach(),
                    ln.bias.detach(), ln.eps)
            stages = []
            for i in range(self._num_stages()):
                blocks = [_KBlock(blk) for blk in net.layers[i].blocks]
                down = _KDown(net.layers[i].downsample) if i + 1 < self._num_stages() else None
                norm = getattr(post, f"norm{i}", None) if i in self.return_indices else None
                stages.append((blocks, down, (norm.weight.detach(), norm.bias.detach(), norm.eps) if norm is not None else None))
            return stem, stages
        return derived.cached(self, "kernel_weights", list(self.parameters()) + list(self.buffers()), build)

    def forward_tokens(self, x: Tensor) -> Dict[str, Tensor]:
        """The backbone on ``x`` (b, 3, H, W) -> {"layers.{i}.blocks": (b, C, h, w)} for i in return_indices, each a
        channels-last view (strides (h*w*C, 1, w*C, C)) of its own (b, h*w, C) token buffer; the values of forward() in torch.
        No host synchronisation."""
        if not self.tokens_supported(x):
            raise RuntimeError("forward_tokens: this call needs forward() (see tokens_supported)")
        (stem_w, stem_b, ln_w, ln_b, eps), stages = self._kernel_weights()
        hw = ((x.shape[2] + 3) // 4, (x.shape[3] + 3) // 4)
        t = cabi.focalnet_stem(x, stem_w, stem_b, ln_w, ln_b, eps)
        feats = {}
        for i, (blocks, down, norm) in enumerate(stages):
            for k in blocks:
                t = self._block_tokens(k, t, hw)
            if norm is not None:
                feats[i] = (cabi.layernorm_tokens(t, *norm), hw)
            if down is not None:
                t = cabi.conv2d_f16x3(t, hw, cabi.pow2_scale(t, 12), *down.w, down.b, 1, 3, 2)
                t = cabi.layernorm_tokens(t, *down.ln)
                hw = ((hw[0] + 1) // 2, (hw[1] + 1) // 2)
        return token_maps(feats, self.return_indices, lambda i: f"layers.{i}.blocks")

    @staticmethod
    def _block_tokens(k: _KBlock, t: Tensor, hw: Tuple[int, int]) -> Tensor:
        # t = t + g1 * norm1(proj(q * h(ctx_all))), then t = t + g2 * norm2(fc2(GELU(fc1(t)))): written over the block input
        C, L = k.C, k.levels
        fo = cabi.gemm_f16x3_ex(t, cabi.pow2_scale(t, 12), *k.wf, k.bf)  # (b, n, 2C + 8): [q | ctx | gates | zeros]
        ctx_all = torch.empty_like(t)
        partials = cabi.focal_context_partials(t.shape[0], hw, C, t.device)
        ctx = fo[..., C:2 * C]
        for level, w in enumerate(k.dw):
            last = level + 1 == L
            ctx = cabi.focal_level_tokens(ctx, fo[..., 2 * C + level:2 * C + level + 1], hw, w, ctx_all, level == 0,
                                          out=not last, partials=partials if last else None)
        cabi.focal_global_context(partials, fo[..., 2 * C + L:2 * C + L + 1], hw, ctx_all, L, k.normalize)
        h = cabi.gemm_f16x3_ex(ctx_all, cabi.pow2_scale(ctx_all, 12), *k.wh, k.bh)
        m = cabi.focal_modulate(fo[..., :C], h, out=h)
        y = cabi.gemm_f16x3_ex(m, cabi.pow2_scale(m, 12), *k.wproj, k.bproj)
        cabi.layernorm_scale_add_tokens_(t, y, *k.ln1[:2], k.g1, k.ln1[2])
        u = cabi.gemm_f16x3_ex(t, cabi.pow2_scale(t, 12), *k.w1, k.b1)
        y = cabi.gemm_f16x3_ex(u, cabi.pow2_scale(u, 12), *k.w2, k.b2, act=cabi.ACT_GELU)
        return cabi.layernorm_scale_add_tokens_(t, y, *k.ln2[:2], k.g2, k.ln2[2])
