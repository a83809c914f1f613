"""Drop-in mirror of the DECODER HALF of the reference's ``models/bricks/salience_transformer.py`` (SURVEY.md 8(f)-1).

``SalienceTransformerDecoderLayer`` (:498-588) and ``SalienceTransformerDecoder`` (:591-674) with the reference's
constructor arguments, sub-module / parameter names and ``forward`` signatures, ``MLP`` (models/bricks/basic.py:7-26),
``get_sine_pos_embed`` (position_encoding.py:105-135) and ``inverse_sigmoid`` (util/misc.py:31-35): a reference
``state_dict`` loads strictly.

Where the time of the decoder is, and what runs on the hand-written kernels:

* ``value`` (the encoder memory) is the same tensor for all six layers (:646), so -- as in the encoder -- the six
  ``cross_attn.value_proj`` GEMMs over all Nv tokens (17.5 GFLOP each at config 2) are ONE tensor-core GEMM with the
  concatenated weights (activation-stationary 3xFP16 kernel), masked rows zeroed once;
* the cross-attention core is the fused sampling kernel with 4-d reference BOXES (softmax + ``ref_xy + off / P * ref_wh / 2``
  + bilinear gather in one launch, ``sdetr_msda_fused_forward_boxes``);
* residual + LayerNorm are the fused row kernel;
* everything that touches only the ~900 (+ denoising) queries -- self-attention, FFN, heads, the sine embedding of the
  reference boxes -- is launch-latency bound; it stays on library kernels (cuBLAS / ``nn.MultiheadAttention``'s fused path) and
  is meant to be replayed from a CUDA graph together with the encoder half.
The training path (autograd) follows the reference's op chain around ``MultiScaleDeformableAttnFunction``.
"""
from __future__ import annotations

import copy
import math
from typing import Optional

import torch
from torch import Tensor, nn
from torch.nn import functional as F

from . import cabi, derived, gemm
from .ms_deform_attn import MultiScaleDeformableAttention


def inverse_sigmoid(x: Tensor, eps: float = 1e-3) -> Tensor:
    """util/misc.py:31-35."""
    x = x.clamp(min=0, max=1)
    return torch.log(x.clamp(min=eps) / (1 - x).clamp(min=eps))


class MLP(nn.Module):
    """models/bricks/basic.py:7-26 (``layers`` ModuleList of Linear, ReLU between)."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))
        for layer in self.layers:
            nn.init.xavier_uniform_(layer.weight)
            nn.init.constant_(layer.bias, 0.0)

    def forward(self, x):
        grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))
        for i, layer in enumerate(self.layers):
            if grad or not x.is_cuda:
                x = F.relu(layer(x)) if i < self.num_layers - 1 else layer(x)
            else:  # ReLU of the previous layer fused into this GEMM's operand load
                x = gemm.linear(x, layer.weight, layer.bias, relu_input=i > 0)
        return x


def get_sine_pos_embed(pos_tensor: Tensor, num_pos_feats: int = 128, temperature: int = 10000, scale: float = 2 * math.pi,
                       exchange_xy: bool = True) -> Tensor:
    """position_encoding.py:105-135: (..., 2n) -> (..., n * num_pos_feats), [pos(y), pos(x), pos(w), pos(h)] order."""
    dim_t = torch.arange(num_pos_feats, dtype=torch.float32, device=pos_tensor.device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / num_pos_feats)
    pos_res = pos_tensor.unsqueeze(-1) * scale / dim_t
    pos_res = torch.stack((pos_res[..., 0::2].sin(), pos_res[..., 1::2].cos()), dim=-1).flatten(-2)
    if exchange_xy:
        index = torch.cat([torch.arange(1, -1, -1, device=pos_res.device), torch.arange(2, pos_res.shape[-2], device=pos_res.device)])
        pos_res = torch.index_select(pos_res, -2, index)
    return pos_res.view(*pos_tensor.shape[:-1], -1)


class SalienceTransformerDecoderLayer(nn.Module):
    def __init__(self, embed_dim=256, d_ffn=1024, n_heads=8, dropout=0.1, activation=nn.ReLU(inplace=True), n_levels=4,
                 n_points=4):
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = n_heads
        self.cross_attn = MultiScaleDeformableAttention(embed_dim, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(embed_dim)
        self.self_attn = nn.MultiheadAttention(embed_dim, n_heads, dropout=dropout, batch_first=True)
        self.dropout2 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(embed_dim)
        self.linear1 = nn.Linear(embed_dim, d_ffn)
        self.activation = activation
        self.dropout3 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, embed_dim)
        self.dropout4 = nn.Dropout(dropout)
        self.norm3 = nn.LayerNorm(embed_dim)
        self.init_weights()

    def init_weights(self):
        nn.init.xavier_uniform_(self.self_attn.in_proj_weight)
        nn.init.xavier_uniform_(self.self_attn.out_proj.weight)
        nn.init.xavier_uniform_(self.linear1.weight)
        nn.init.xavier_uniform_(self.linear2.weight)

    @staticmethod
    def with_pos_embed(tensor, pos):
        return tensor if pos is None else tensor + pos

    def forward_ffn(self, tgt):
        tgt2 = self.linear2(self.dropout3(self.activation(self.linear1(tgt))))
        return self.norm3(tgt + self.dropout4(tgt2))

    def forward(self, query, query_pos, reference_points, value, spatial_shapes, level_start_index, self_attn_mask=None,
                key_padding_mask=None):
        """Reference signature and op order (:552-588): self-attention, cross-attention, FFN, post-norm each."""
        x = self.with_pos_embed(query, query_pos)
        query2 = self.self_attn(query=x, key=x, value=query, attn_mask=self_attn_mask)[0]
        query = self.norm2(query + self.dropout2(query2))
        query2 = self.cross_attn(query=self.with_pos_embed(query, query_pos), reference_points=reference_points, value=value,
                                 spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                                 key_padding_mask=key_padding_mask)
        query = self.norm1(query + self.dropout1(query2))
        return self.forward_ffn(query)

    def forward_fast(self, query, query_pos, reference_points, vbuf, v_bstride, v_tstride, v_off, num_value, spatial_shapes,
                     level_start_index, self_attn_mask=None):
        """Inference: same math on an already projected value buffer (this layer's column slice of the 6-layer GEMM)."""
        x = query + query_pos
        query2 = self.self_attn(query=x, key=x, value=query, attn_mask=self_attn_mask, need_weights=False)[0]
        query = cabi.add_layernorm(query.contiguous(), query2.contiguous(), self.norm2.weight, self.norm2.bias, self.norm2.eps)
        a = self.cross_attn.forward_projected((query + query_pos).contiguous(), reference_points.contiguous(), vbuf, v_bstride,
                                              v_tstride, v_off, num_value, spatial_shapes, level_start_index, None, 0)
        query = cabi.add_layernorm(query, a, self.norm1.weight, self.norm1.bias, self.norm1.eps, out=query)
        h = gemm.linear(query, self.linear1.weight, self.linear1.bias)
        f = gemm.linear(h, self.linear2.weight, self.linear2.bias, relu_input=True)
        return cabi.add_layernorm(query, f, self.norm3.weight, self.norm3.bias, self.norm3.eps, out=query)


class SalienceTransformerDecoder(nn.Module):
    def __init__(self, decoder_layer, num_layers, num_classes):
        super().__init__()
        self.embed_dim = decoder_layer.embed_dim
        self.num_layers = num_layers
        self.num_classes = num_classes
        self.layers = nn.ModuleList([copy.deepcopy(decoder_layer) for _ in range(num_layers)])
        self.ref_point_head = MLP(2 * self.embed_dim, self.embed_dim, self.embed_dim, 2)
        self.class_head = nn.ModuleList([nn.Linear(self.embed_dim, num_classes) for _ in range(num_layers)])
        self.bbox_head = nn.ModuleList([MLP(self.embed_dim, self.embed_dim, 4, 3) for _ in range(num_layers)])
        self.norm = nn.LayerNorm(self.embed_dim)
        self.init_weights()

    def init_weights(self):
        for layer in self.layers:
            if hasattr(layer, "init_weights"):
                layer.init_weights()
        bias_value = -math.log((1 - 0.01) / 0.01)
        for class_head in self.class_head:
            nn.init.constant_(class_head.bias, bias_value)
        for bbox_head in self.bbox_head:
            nn.init.constant_(bbox_head.layers[-1].weight, 0.0)
            nn.init.constant_(bbox_head.layers[-1].bias, 0.0)

    def _value_projection(self):
        ws = [l.cross_attn.value_proj.weight for l in self.layers]
        bs = [l.cross_attn.value_proj.bias for l in self.layers]
        return derived.cached(self, "value_projection", ws + bs, lambda: (torch.cat(ws, 0).contiguous(), torch.cat(bs, 0).contiguous()))

    def forward(self, query, reference_points, value, spatial_shapes, level_start_index, valid_ratios, key_padding_mask=None,
                attn_mask=None):
        """Reference signature (:628-674) -> (outputs_classes (layers,b,nq,classes), outputs_coords (layers,b,nq,4))."""
        outputs_classes, outputs_coords = [], []
        valid_ratio_scale = torch.cat([valid_ratios, valid_ratios], -1)[:, None]
        grad = torch.is_grad_enabled() and (query.requires_grad or value.requires_grad or
                                            any(p.requires_grad for p in self.parameters()))
        fast = not grad and value.is_cuda
        if fast:
            b, nv, c = value.shape
            value = value.contiguous()
            wv, bv = self._value_projection()
            vbuf = gemm.linear(value, wv, bv)  # all layers' cross_attn.value_proj in one GEMM (value never changes, :646)
            wide = vbuf.shape[-1]
            if key_padding_mask is not None:
                cabi.zero_masked_rows_(vbuf, wide, wide, key_padding_mask.to(torch.uint8).contiguous(), b * nv)
            spatial_shapes = spatial_shapes.to(torch.int64).contiguous()
            level_start_index = level_start_index.to(torch.int64).contiguous()
            query = query.contiguous()
        for layer_idx, layer in enumerate(self.layers):
            reference_points_input = reference_points.detach()[:, :, None] * valid_ratio_scale
            query_sine_embed = get_sine_pos_embed(reference_points_input[:, :, 0, :])
            query_pos = self.ref_point_head(query_sine_embed)
            if fast:
                query = layer.forward_fast(query, query_pos, reference_points_input, vbuf, nv * wide, wide, layer_idx * c, nv,
                                           spatial_shapes, level_start_index, self_attn_mask=attn_mask)
            else:
                query = layer(query=query, query_pos=query_pos, reference_points=reference_points_input, value=value,
                              spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                              key_padding_mask=key_padding_mask, self_attn_mask=attn_mask)
            normed = self.norm(query)
            output_class = self.class_head[layer_idx](normed)
            output_coord = (self.bbox_head[layer_idx](normed) + inverse_sigmoid(reference_points)).sigmoid()
            outputs_classes.append(output_class)
            outputs_coords.append(output_coord)
            if layer_idx == self.num_layers - 1:
                break
            reference_points = (self.bbox_head[layer_idx](query) + inverse_sigmoid(reference_points.detach())).sigmoid()
        return torch.stack(outputs_classes), torch.stack(outputs_coords)
