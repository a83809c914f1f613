"""Drop-in mirror of the ENCODER HALF of the reference's ``models/bricks/salience_transformer.py``.

Same class names, constructor arguments, sub-module / parameter names and ``forward`` signatures
(``MaskPredictor`` :16-47, ``SalienceTransformerEncoderLayer`` :298-396, ``SalienceTransformerEncoder``
:399-497, the encoder half of ``SalienceTransformer`` :50-183), so a reference ``state_dict`` loads
(``strict=False`` skips the decoder keys) and reference configs can instantiate these classes in place
of the originals.  The decoder half (:194-295, :500-674) is out of scope for this round (SURVEY.md 8(f)-1).

How the path is laid out for an H100 (none of this is a translation of the reference's op chain):

* one ``EncoderPlan`` per batch geometry holds everything derived from the padding masks (token budgets,
  level tables, valid ratios, keep mask).  Building it costs ONE host round trip; the reference syncs
  ~40 times per forward (SURVEY.md section 3a).  With a plan the forward is sync-free and CUDA-graph
  capturable.
* the salience filter is a single C-ABI call after the coarse-to-fine score loop;
* ``value`` never changes across encoder layers (:452), so the six ``value_proj`` GEMMs are ONE GEMM over
  the concatenated weights, the padded rows are zeroed once, and every layer samples its column slice;
* per layer: one fused four-way gather, one GEMM for offsets|logits, one fused
  softmax+locations+sampling kernel (spatially tiled processing order), fused residual+LayerNorm,
  in-place prefix-limited scatter.  At C = 256 (head_dim 32) the 300-token pre-attention is three fused kernels and the
  FFN is one; other widths run the pre-attention's projections / attention on cuBLAS / SDPA and the FFN as two GEMMs.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn
from torch.nn import functional as F

from . import cabi, derived, gemm
from .channel_mapper import tokens_of
from .ms_deform_attn import MultiScaleDeformableAttention

PREDICTOR_SMALL_ROWS = 4096  # score modulation + MaskPredictor of a level with at most this many token rows as two fp32
# kernels (csrc/predictor_small.cu) instead of ~15 latency-bound launches; 0 = never
TILE_CELL_PX = 64   # edge (image pixels) of the spatial cells that define the MSDA processing order
MSDA_SCHEDULE = 1   # 0 = query-major, 1 = head-major chunks (see include/sdetr_b200.h)


class MaskPredictor(nn.Module):
    """Per-token salience score (reference :16-47): LN -> Linear -> GELU, global half = token mean."""

    def __init__(self, in_dim, h_dim):
        super().__init__()
        self.h_dim = h_dim
        self.layer1 = nn.Sequential(nn.LayerNorm(in_dim), nn.Linear(in_dim, h_dim), nn.GELU())
        self.layer2 = nn.Sequential(nn.Linear(h_dim, h_dim // 2), nn.GELU(), nn.Linear(h_dim // 2, h_dim // 4),
                                    nn.GELU(), nn.Linear(h_dim // 4, 1))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                nn.init.constant_(m.bias, 0)

    def forward(self, x):
        z = self.layer1(x)
        half = self.h_dim // 2
        z = torch.cat([z[..., :half], z[..., half:].mean(dim=1, keepdim=True).expand(-1, z.shape[1], -1)], dim=-1)
        return self.layer2(z)

    def transposed_weights(self):
        """(W1^T, b1, W2a^T, b2a, W2b^T, b2b, w2c, b2c) with the weights in (in, out) layout, cached per parameter version
        (sdetr_mask_predictor_level streams weight rows)."""
        lins = [self.layer1[1], self.layer2[0], self.layer2[2], self.layer2[4]]
        return derived.cached(self, "transposed_weights", [t for m in lins for t in (m.weight, m.bias)], lambda: (
            lins[0].weight.detach().t().contiguous(), lins[0].bias.detach(), lins[1].weight.detach().t().contiguous(),
            lins[1].bias.detach(), lins[2].weight.detach().t().contiguous(), lins[2].bias.detach(),
            lins[3].weight.detach().reshape(-1).contiguous(), lins[3].bias.detach()))

    def forward_fast(self, x):
        """Inference: same math; projections on the tensor cores, GELUs fused into the next GEMM's operand load,
        LayerNorm by the fused kernel, global half written in place instead of split/expand/cat."""
        ln, fc = self.layer1[0], self.layer1[1]
        x = x if x.is_contiguous() else x.contiguous()
        z = gemm.linear(cabi.add_layernorm(x, None, ln.weight, ln.bias, ln.eps), fc.weight, fc.bias)
        half = self.h_dim // 2
        if z.dim() == 3 and z.is_contiguous() and self.h_dim % 8 == 0 and self.h_dim <= 1024:
            cabi.gelu_colmean_(z, half)  # GELU + global half = token mean, broadcast in place (:40-45), two launches
        else:
            z = F.gelu(z)
            z[..., half:] = z[..., half:].mean(dim=1, keepdim=True)
        z = gemm.linear(z, self.layer2[0].weight, self.layer2[0].bias)
        z = gemm.linear(z, self.layer2[2].weight, self.layer2[2].bias, input_act="gelu")
        return gemm.linear(z, self.layer2[4].weight, self.layer2[4].bias, input_act="gelu")


class PositionEmbeddingLearned(nn.Module):
    """Learned row/col embedding used as the encoder's background embedding (position_encoding.py:68-95)."""

    def __init__(self, num_embeddings: int = 50, num_pos_feats: int = 256):
        super().__init__()
        self.row_embed = nn.Embedding(num_embeddings, num_pos_feats)
        self.col_embed = nn.Embedding(num_embeddings, num_pos_feats)
        nn.init.uniform_(self.row_embed.weight)
        nn.init.uniform_(self.col_embed.weight)

    def forward(self, mask: Tensor):
        h, w = mask.shape[-2:]
        x = self.col_embed.weight[:w][None].expand(h, -1, -1)
        y = self.row_embed.weight[:h][:, None].expand(-1, w, -1)
        return torch.cat([x, y], -1).permute(2, 0, 1)[None].expand(mask.shape[0], -1, -1, -1)


# ------------------------------------------------------------------------------------------------------------
@dataclass
class EncoderPlan:
    """Everything the path derives from the padding masks (one host sync to build, none to use)."""
    shapes_list: List[Tuple[int, int]]
    spatial_shapes: Tensor      # (L,2) int64, device
    level_start_index: Tensor   # (L,) int64, device
    level_start: List[int]
    level_size: List[int]
    level_width: List[int]
    level_stride: List[int]     # image pixels per token, for the processing-order cells
    mask_flat: Tensor           # (b,Nv) bool
    mask_u8: Tensor             # (b,Nv) uint8
    keep: Tensor                # (b,Nv,1) float: ~padding & proposal-valid (base_transformer.py:100-108)
    valid_ratios: Tensor        # (b,L,2)
    level_token_nums: List[int]
    focus_token_nums: Tensor    # (b,) int32, device
    focus_host: List[int]
    num_selected: int           # K
    layer_num_query: List[int]
    scratch: Dict[str, Tensor] = field(default_factory=dict)


class UpsampleBilinearAC(torch.autograd.Function):
    """``F.interpolate(x, size, mode="bilinear", align_corners=True)`` with a deterministic backward
    (``sdetr_upsample_bilinear_ac_backward``, gather form).  torch's CUDA backward of the op accumulates with atomics and
    raises under ``torch.use_deterministic_algorithms(True)``; the forward is the same torch call, so its bits do not change."""

    @staticmethod
    def forward(ctx, x, size):
        ctx.in_hw = tuple(x.shape[-2:])
        return F.interpolate(x, size=size, mode="bilinear", align_corners=True)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad):
        return cabi.upsample_bilinear_ac_backward(grad.contiguous(), *ctx.in_hw), None


def flatten_levels(xs: Sequence[Tensor]) -> Tensor:
    """(b,[C],H_l,W_l) per level -> (b,Nv,[C]) tokens (base_transformer.py:21-26)."""
    y = torch.cat([e.flatten(-2) for e in xs], -1)
    return y.transpose(1, 2).contiguous() if y.ndim == 3 else y


class SalienceTransformerEncoderLayer(nn.Module):
    def __init__(self, embed_dim=256, d_ffn=1024, dropout=0.1, n_heads=8, activation=nn.ReLU(inplace=True), n_levels=4,
                 n_points=4, topk_sa=300):
        super().__init__()
        self.embed_dim = embed_dim
        self.topk_sa = topk_sa
        self.n_heads = n_heads
        self.pre_attention = nn.MultiheadAttention(embed_dim, n_heads, dropout, batch_first=True)
        self.pre_dropout = nn.Dropout(dropout)
        self.pre_norm = nn.LayerNorm(embed_dim)
        self.self_attn = MultiScaleDeformableAttention(embed_dim, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(embed_dim)
        self.linear1 = nn.Linear(embed_dim, d_ffn)
        self.activation = activation
        self.dropout2 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, embed_dim)
        self.dropout3 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(embed_dim)
        self.init_weights()

    def init_weights(self):
        nn.init.xavier_uniform_(self.pre_attention.in_proj_weight)
        nn.init.xavier_uniform_(self.pre_attention.out_proj.weight)
        nn.init.xavier_uniform_(self.linear1.weight)
        nn.init.xavier_uniform_(self.linear2.weight)

    # -- reference-signature forward (autograd friendly; used for training) ---------------------------------
    def forward(self, query, query_pos, value, reference_points, spatial_shapes, level_start_index,
                query_key_padding_mask=None, score_tgt=None, foreground_pre_layer=None):
        mc = score_tgt.max(-1)[0] * foreground_pre_layer
        top = cabi.topk_desc(mc.detach().float().contiguous(), min(self.topk_sa, mc.shape[1]))
        ix = top.unsqueeze(-1).expand(-1, -1, self.embed_dim)
        t, tp = torch.gather(query, 1, ix), torch.gather(query_pos, 1, ix)
        x = t + tp
        t = self.pre_norm(t + self.pre_dropout(self.pre_attention(x, x, t)[0]))
        query = query.scatter(1, ix, t)
        a = self.self_attn(query=query + query_pos, reference_points=reference_points, value=value,
                           spatial_shapes=spatial_shapes, level_start_index=level_start_index,
                           key_padding_mask=query_key_padding_mask)
        query = self.norm1(query + self.dropout1(a))
        f = self.linear2(self.dropout2(self.activation(self.linear1(query))))
        return self.norm2(query + self.dropout3(f))

    # -- inference fast path ------------------------------------------------------------------------------------
    def _mha_views(self):
        """Views of in_proj_{weight,bias}: [q|k] rows and [v] rows."""
        w, bias, c = self.pre_attention.in_proj_weight, self.pre_attention.in_proj_bias, self.embed_dim
        return derived.cached(self, "mha_views", (w, bias), lambda: (
            w.detach()[:2 * c], bias.detach()[:2 * c], w.detach()[2 * c:], bias.detach()[2 * c:]))

    def _mha_transposed(self):
        """in_proj_weight^T (C,3C) and out_proj.weight^T (C,C), cached per parameter version (the fused pre-attention
        kernels stream weight rows of the (in, out) layout)."""
        w, wo = self.pre_attention.in_proj_weight, self.pre_attention.out_proj.weight
        return derived.cached(self, "mha_transposed", (w, wo), lambda: (w.detach().t().contiguous(), wo.detach().t().contiguous()))

    def _pre_attention_fast(self, q, qp, mc, qs=None):
        """Top-k salient tokens -> MHA -> LN -> scatter (reference :366-379).  C = 256, head_dim = 32 (every reference
        config): three fused fp32 kernels (csrc/mha_small.cu); other geometries: library projections / SDPA between
        the fused gather / residual+LN / scatter kernels."""
        b, nq, c = q.shape
        k = min(self.topk_sa, nq)
        top = cabi.topk_desc(mc, k)
        if c == 256 and c // self.n_heads == 32 and k <= 448:  # attention kernel: K/V/P in smem
            w_in_t, w_out_t = self._mha_transposed()
            t, qkv = cabi.mha_in_proj(q, qp, top, w_in_t, self.pre_attention.in_proj_bias)
            o = cabi.attention_qkv(qkv, self.n_heads)
            cabi.mha_out_proj_ln_scatter_(q, o, t, w_out_t, self.pre_attention.out_proj.bias, self.pre_norm.weight,
                                          self.pre_norm.bias, self.pre_norm.eps, top, qp if qs is not None else None, qs)
            return q, qs, top
        t, x = cabi.rows_gather_add(q, qp, top)           # t = q[top], x = t + qp[top]
        wqk, bqk, wv, bv = self._mha_views()
        h, d = self.n_heads, c // self.n_heads
        qk = F.linear(x, wqk, bqk).view(b, k, 2, h, d)
        v = F.linear(t, wv, bv).view(b, k, h, d)
        o = F.scaled_dot_product_attention(qk[:, :, 0].transpose(1, 2), qk[:, :, 1].transpose(1, 2), v.transpose(1, 2))
        o = o.transpose(1, 2).reshape(b, k, c)
        o = F.linear(o, self.pre_attention.out_proj.weight, self.pre_attention.out_proj.bias)
        t = cabi.add_layernorm(t, o, self.pre_norm.weight, self.pre_norm.bias, self.pre_norm.eps)
        cabi.rows_scatter_(q, top, t)  # q is this layer's private gather buffer
        return q, None, top

    def forward_fast(self, q, qp, mc, ref_q, vbuf, v_bstride, v_tstride, v_off, num_value, spatial_shapes,
                     level_start_index, order=None, qs=None):
        """``qs``: optional q + qp buffer (from the gather); the fused pre-attention keeps its rewritten rows current."""
        q, qs, top = self._pre_attention_fast(q, qp, mc, qs)
        s = self.self_attn.sample_projected(qs if qs is not None else q + qp, ref_q, vbuf, v_bstride, v_tstride, v_off, num_value,
                                            spatial_shapes, level_start_index, order, MSDA_SCHEDULE)
        op = self.self_attn.output_proj
        if self.embed_dim == 256 and q.is_contiguous() and gemm.f16x3_route(s, op.weight, op.bias):
            # output projection, residual and norm1 in one launch, bit for bit the two below
            w_hi, w_lo, w_scale = gemm.split_weight_f16(op.weight)
            cabi.gemm_f16x3_add_layernorm_(q, gemm._rows(s), w_hi, w_lo, w_scale, op.bias, self.norm1.weight, self.norm1.bias,
                                           self.norm1.eps)
        else:
            q = cabi.add_layernorm(q, gemm.linear(s, op.weight, op.bias), self.norm1.weight, self.norm1.bias, self.norm1.eps, out=q)
        rows = q.shape[0] * q.shape[1]
        relu = isinstance(self.activation, nn.ReLU)
        if (relu and self.embed_dim == 256 and self.linear1.out_features % 128 == 0 and gemm.MODE == "auto" and
                gemm.OWN_KERNEL == "f16x3" and rows > gemm.SMALL_M and q.is_contiguous()):
            return cabi.ffn_fused_layernorm(q, gemm.split_weight_f16(self.linear1.weight), self.linear1.bias,
                                            gemm.split_weight_f16(self.linear2.weight), self.linear2.bias, self.norm2.weight,
                                            self.norm2.bias, self.norm2.eps, out=q)
        h = gemm.linear(q, self.linear1.weight, self.linear1.bias)
        if relu:
            f = gemm.linear(h, self.linear2.weight, self.linear2.bias, relu_input=True)  # ReLU fused into the operand split
        else:  # any other activation module of the reference's constructor argument
            f = gemm.linear(self.activation(h), self.linear2.weight, self.linear2.bias)
        return cabi.add_layernorm(q, f, self.norm2.weight, self.norm2.bias, self.norm2.eps, out=q)


class SalienceTransformerEncoder(nn.Module):
    def __init__(self, encoder_layer: nn.Module, num_layers: int = 6, max_num_embedding=200):
        super().__init__()
        self.layers = nn.ModuleList([copy.deepcopy(encoder_layer) for _ in range(num_layers)])
        self.num_layers = num_layers
        self.embed_dim = encoder_layer.embed_dim
        self.background_embedding = PositionEmbeddingLearned(max_num_embedding, num_pos_feats=self.embed_dim // 2)
        self.enhance_mcsp: Optional[nn.Module] = None  # injected by SalienceTransformer (reference :79)
        for layer in self.layers:
            layer.init_weights()

    @staticmethod
    def get_reference_points(spatial_shapes, valid_ratios, device):
        """(b,Nv,L,2) table of the reference (:417-432); the fast path never materialises it (the gather
        kernel recomputes the needed rows), this exists for API parity and the training path."""
        refs = []
        for lvl, (h, w) in enumerate(spatial_shapes.tolist() if torch.is_tensor(spatial_shapes) else spatial_shapes):
            ys = torch.arange(h, dtype=torch.float32, device=device) + 0.5
            xs = torch.arange(w, dtype=torch.float32, device=device) + 0.5
            ry = ys[None, :, None].expand(1, h, w).reshape(1, -1) / (valid_ratios[:, None, lvl, 1] * h)
            rx = xs[None, None, :].expand(1, h, w).reshape(1, -1) / (valid_ratios[:, None, lvl, 0] * w)
            refs.append(torch.stack((rx, ry), -1))
        return torch.cat(refs, 1)[:, :, None] * valid_ratios[:, None]

    def _value_projection(self):
        """[6*C, C] weight / [6*C] bias of all layers' value_proj (rebuilt when any of them changes)."""
        ws = [l.self_attn.value_proj.weight for l in self.layers]
        bs = [l.self_attn.value_proj.bias for l in self.layers]
        return derived.cached(self, "value_projection", ws + bs, lambda: (torch.cat(ws, 0).contiguous(), torch.cat(bs, 0).contiguous()))

    def project_values(self, tokens: Tensor, mask_u8: Tensor) -> Tensor:
        """(b,Nv,C) value tokens -> (b,Nv,layers*C): every layer's value_proj in ONE GEMM (the value tokens never
        change across layers, reference :452), padded rows zeroed (ms_deform_attn.py:318-319)."""
        b, nv, _ = tokens.shape
        wv, bv = self._value_projection()
        vbuf = gemm.linear(tokens, wv, bv)
        wide = vbuf.shape[-1]
        cabi.zero_masked_rows_(vbuf, wide, wide, mask_u8, b * nv)
        return vbuf

    def forward(self, query, spatial_shapes, level_start_index, valid_ratios, query_pos=None,
                query_key_padding_mask=None, foreground_score=None, focus_token_nums=None, foreground_inds=None,
                multi_level_masks=None, query_orders=None, value_buffer=None, focus_host=None):
        """Reference signature (:434-447) + optional ``query_orders`` (per-layer int32 processing orders) and ``focus_host`` (the
        focus counts as host ints: the training path then needs no device -> host copy and can be captured in a CUDA graph).

        query/query_pos (b,Nv,C); foreground_inds: list of (b,Nq_j) int64 (prefix views of one selected_inds);
        focus_token_nums (b,) int; -> encoder memory (b,Nv,C)."""
        if torch.is_grad_enabled() and (query.requires_grad or any(p.requires_grad for p in self.parameters())):
            return self._forward_autograd(query, spatial_shapes, level_start_index, valid_ratios, query_pos,
                                          query_key_padding_mask, foreground_score, focus_token_nums, foreground_inds,
                                          multi_level_masks, focus_host)
        b, nv, c = query.shape
        L = spatial_shapes.shape[0]
        M = self.layers[0].self_attn.num_heads
        query = query.contiguous()  # the reference hands over a transposed view (base_transformer.py:21-26)
        mask_u8 = query_key_padding_mask.to(torch.uint8).contiguous()
        focus = focus_token_nums.to(torch.int32).contiguous()
        # one GEMM for the value projections of all layers; zero the padded rows once
        vbuf = value_buffer if value_buffer is not None else self.project_values(query, mask_u8)
        wide = vbuf.shape[-1]
        out = query.clone()  # `value` stays the original tokens (:452); `out` is updated in place
        spatial_shapes = spatial_shapes.to(torch.int64).contiguous()
        level_start_index = level_start_index.to(torch.int64).contiguous()
        pos = query_pos.contiguous()
        fg = foreground_score.contiguous()
        vr = valid_ratios.contiguous()
        inds = None
        for j, layer in enumerate(self.layers):
            inds = foreground_inds[j]
            nq = inds.shape[1]
            q, qp, fq, rq, qs = cabi.token_gather(out, pos, fg, vr, inds, spatial_shapes, level_start_index, nq, want_sum=True)
            w, bw = self.enhance_mcsp.weight, self.enhance_mcsp.bias
            if w.shape[0] <= 128 and gemm.f16x3_route(q, w, bw):  # class scores and their row max in one launch, bit for bit
                w_hi, w_lo, w_scale = gemm.split_weight_f16(w)
                mc = cabi.gemm_f16x3_rowmax(gemm._rows(q), w_hi, w_lo, w_scale, bw, fq).view(fq.shape)
            else:
                mc = cabi.class_max_times_fg(gemm.linear(q, w, bw), fq)
            q = layer.forward_fast(q, qp, mc, rq, vbuf, nv * wide, wide, j * c, nv, spatial_shapes,
                                   level_start_index, None if query_orders is None else query_orders[j], qs=qs)
            cabi.token_scatter_(out, q, inds, focus)
        if multi_level_masks is not None:
            cabi.background_embed_(out, mask_u8, inds, self.background_embedding.row_embed.weight,
                                   self.background_embedding.col_embed.weight, spatial_shapes, level_start_index,
                                   shapes_host=[tuple(m.shape[-2:]) for m in multi_level_masks])
        return out

    def _forward_autograd(self, query, spatial_shapes, level_start_index, valid_ratios, query_pos,
                          query_key_padding_mask, foreground_score, focus_token_nums, foreground_inds, multi_level_masks,
                          focus_host=None):
        """Training path: torch autograd around the custom MSDA Function (forward + backward kernels).  With the level shapes
        (from the masks) and ``focus_host`` known on the host there is no device -> host copy in it."""
        b, nv, c = query.shape
        shapes = [tuple(m.shape[-2:]) for m in multi_level_masks] if multi_level_masks is not None else spatial_shapes
        ref = self.get_reference_points(shapes, valid_ratios, query.device)
        L = ref.shape[2]
        value = output = query
        focus = list(focus_host) if focus_host is not None else focus_token_nums.tolist()
        inds = None
        for j, layer in enumerate(self.layers):
            inds = foreground_inds[j]
            nq = inds.shape[1]
            ix = inds.unsqueeze(-1).expand(-1, -1, c)
            q, qp = torch.gather(output, 1, ix), torch.gather(query_pos, 1, ix)
            fq = torch.gather(foreground_score, 1, inds)
            rq = torch.gather(ref.view(b, nv, -1), 1, inds.unsqueeze(-1).expand(-1, -1, L * 2)).view(b, nq, L, 2)
            q = layer(q, qp, value, rq, spatial_shapes, level_start_index, query_key_padding_mask, self.enhance_mcsp(q), fq)
            rows = []
            for i in range(b):
                n = min(int(focus[i]), nq)
                rows.append(output[i].scatter(0, inds[i, :n].unsqueeze(-1).expand(-1, c), q[i, :n]))
            output = torch.stack(rows)
        if multi_level_masks is not None:
            bg = torch.cat([self.background_embedding(m).flatten(2).transpose(1, 2) for m in multi_level_masks], 1).clone()
            bg.scatter_(1, inds.unsqueeze(-1).expand(-1, -1, c), 0)
            output = output + bg * (~query_key_padding_mask).unsqueeze(-1)
        return output


class SalienceTransformer(nn.Module):
    """Encoder half of the reference ``SalienceTransformer`` (:50-183): salience filter + encoder.

    Constructor signature follows the reference (:51-61); ``neck`` / ``decoder`` may be ``None`` (they are
    outside this round's path).  Parameters of the path keep the reference names: ``level_embeds``,
    ``enc_output``, ``enc_output_norm``, ``alpha``, ``level_filter_ratio``, ``layer_filter_ratio``,
    ``encoder_class_head``, ``enc_mask_predictor``, ``encoder.*``."""

    def __init__(self, encoder: nn.Module, neck: Optional[nn.Module] = None, decoder: Optional[nn.Module] = None,
                 num_classes: int = 91, num_feature_levels: int = 4, two_stage_num_proposals: int = 900,
                 level_filter_ratio: Tuple = (0.25, 0.5, 1.0, 1.0),
                 layer_filter_ratio: Tuple = (1.0, 0.8, 0.6, 0.6, 0.4, 0.2), level_strides: Sequence[int] = (8, 16, 32, 64)):
        super().__init__()
        self.embed_dim = encoder.embed_dim
        self.num_feature_levels = num_feature_levels
        self.two_stage_num_proposals = two_stage_num_proposals
        self.num_classes = num_classes
        self.level_strides = list(level_strides)
        self.level_embeds = nn.Parameter(torch.empty(num_feature_levels, self.embed_dim))
        self.enc_output = nn.Linear(self.embed_dim, self.embed_dim)
        self.enc_output_norm = nn.LayerNorm(self.embed_dim)
        self.register_buffer("level_filter_ratio", torch.tensor(level_filter_ratio, dtype=torch.float32))
        self.register_buffer("layer_filter_ratio", torch.tensor(layer_filter_ratio, dtype=torch.float32))
        self.alpha = nn.Parameter(torch.empty(3), requires_grad=True)
        self.encoder = encoder
        self.neck = neck
        self.decoder = decoder
        self.encoder_class_head = nn.Linear(self.embed_dim, num_classes)
        self.encoder.enhance_mcsp = self.encoder_class_head
        self.enc_mask_predictor = MaskPredictor(self.embed_dim, self.embed_dim)
        if decoder is not None:  # decoder half (reference :74-77): only then do these parameters exist in the state_dict
            from .decoder import MLP
            self.tgt_embed = nn.Embedding(two_stage_num_proposals, self.embed_dim)
            self.encoder_bbox_head = MLP(self.embed_dim, self.embed_dim, 4, 3)
        # not a sub-module of the reference transformer (the detector owns it, salience_detr.py:150-176); attach one
        # (``position_encoding.PositionEmbeddingSine``) to let forward_encoder derive the embeddings from the masks
        self.__dict__["position_embedding"] = None
        self.init_weights()

    def init_weights(self):
        import math
        nn.init.normal_(self.level_embeds)
        nn.init.xavier_uniform_(self.enc_output.weight)
        nn.init.constant_(self.enc_output.bias, 0.0)
        nn.init.constant_(self.encoder_class_head.bias, -math.log((1 - 0.01) / 0.01))
        if self.decoder is not None:
            nn.init.normal_(self.tgt_embed.weight)
            nn.init.constant_(self.encoder_bbox_head.layers[-1].weight, 0.0)
            nn.init.constant_(self.encoder_bbox_head.layers[-1].bias, 0.0)
        self.alpha.data.uniform_(-0.3, 0.3)

    def _side_stream(self, device):
        """One side stream per (device, CURRENT stream): forwards captured from different streams must not meet on a shared
        side stream, which would order their value projections one after the other."""
        streams = self.__dict__.setdefault("_side_streams", {})
        key = (str(device), torch.cuda.current_stream(device).cuda_stream)
        if key not in streams:
            streams[key] = torch.cuda.Stream(device=device)
        return streams[key]

    # -- plan ------------------------------------------------------------------------------------------------
    def _ratios_host(self):
        """Host copies of the two ratio buffers (one device read per buffer version, not one per plan)."""
        lv, ly = self.level_filter_ratio, self.layer_filter_ratio
        return derived.cached(self, "ratios_host", (lv, ly), lambda: (lv.detach().float().cpu().numpy().copy(),
                                                                       ly.detach().float().cpu().numpy().copy()))

    @torch.no_grad()
    def make_plan(self, multi_level_masks: Sequence[Tensor]) -> EncoderPlan:
        """Token budgets (:117-121, :161-165), level tables (base_transformer.py:34-56), the proposal keep mask
        (base_transformer.py:74-110) and the normalised coordinates of the sine position embedding from the padding
        masks.  CUDA masks: two launches (``sdetr_mask_plan``) + ONE device->host copy of b*L ints.  CPU masks (host-logic
        tests only): the same arithmetic in torch ops."""
        import numpy as np
        dev = multi_level_masks[0].device
        b = multi_level_masks[0].shape[0]
        if len(multi_level_masks) != self.num_feature_levels:
            raise ValueError(f"{len(multi_level_masks)} feature levels given, model built for {self.num_feature_levels}")
        shapes_list = [tuple(int(s) for s in m.shape[-2:]) for m in multi_level_masks]
        L = len(shapes_list)
        sizes = [h * w for h, w in shapes_list]
        starts = [sum(sizes[:i]) for i in range(L)]
        spatial_shapes = torch.tensor(shapes_list, dtype=torch.int64, device=dev)
        level_start_index = torch.tensor(starts, dtype=torch.int64, device=dev)
        mask_flat = flatten_levels(multi_level_masks)
        mask_u8 = mask_flat.to(torch.uint8).contiguous()
        level_ratio, layer_ratio = self._ratios_host()
        scratch = {}
        if mask_flat.is_cuda:
            pe = getattr(self, "position_embedding", None)
            mp = cabi.mask_plan(mask_u8, shapes_list, level_ratio.tolist(), *((pe.offset, pe.eps, pe.scale) if pe is not None
                                                                              else (-0.5, 1e-6, 2 * 3.141592653589793)))
            focus = mp["focus"]
            focus_np = focus.cpu().numpy()                                               # the one sync
            keep, valid_ratios = mp["keep"].unsqueeze(-1), mp["valid_ratios"]
            scratch["ynorm"], scratch["xnorm"] = mp["ynorm"], mp["xnorm"]
            focus_sum = focus.sum(-1).to(torch.int32).contiguous()
        else:
            valid = torch.stack([(~m).sum((1, 2)) for m in multi_level_masks], -1)       # (b,L) int64
            focus = (valid * self.level_filter_ratio).int()                              # fp32 multiply, truncate
            vr, keep = [], []
            for lvl, m in enumerate(multi_level_masks):
                h, w = shapes_list[lvl]
                vh, vw = (~m[:, :, 0]).sum(1), (~m[:, 0, :]).sum(1)
                vr.append(torch.stack([vw.float() / w, vh.float() / h], -1))
                gy = (torch.arange(h, dtype=torch.float32, device=dev) + 0.5)[None, :, None] / vh[:, None, None]
                gx = (torch.arange(w, dtype=torch.float32, device=dev) + 0.5)[None, None, :] / vw[:, None, None]
                ok = (gy > 0.01) & (gy < 0.99) & (gx > 0.01) & (gx < 0.99) & (0.01 < 0.05 * 2.0 ** lvl < 0.99)
                keep.append((ok & ~m).flatten(1))
            keep = torch.cat(keep, 1).unsqueeze(-1).float()
            valid_ratios = torch.stack(vr, 1).contiguous()
            focus_np = focus.numpy()
            focus_sum = focus.sum(-1).to(torch.int32).contiguous()
        level_token_nums = [int(x) for x in focus_np.max(0)]
        focus_host = [int(x) for x in focus_np.sum(-1)]
        K = sum(level_token_nums)
        layer_nq = [int(x) for x in (np.float32(K) * layer_ratio.astype(np.float32)).astype(np.int64)]  # :164, fp32 multiply
        return EncoderPlan(
            shapes_list=shapes_list, spatial_shapes=spatial_shapes, level_start_index=level_start_index,
            level_start=starts, level_size=sizes, level_width=[w for _, w in shapes_list],
            level_stride=(self.level_strides + [self.level_strides[-1] * 2] * L)[:L], mask_flat=mask_flat,
            mask_u8=mask_u8, keep=keep, valid_ratios=valid_ratios, level_token_nums=level_token_nums,
            focus_token_nums=focus_sum, focus_host=focus_host, num_selected=K, layer_num_query=layer_nq, scratch=scratch)

    def attach_position_embedding(self, module) -> "SalienceTransformer":
        """Attach the detector's position-embedding module WITHOUT registering it as a sub-module (the reference
        transformer's state_dict has no such entry)."""
        self.__dict__["position_embedding"] = module
        return self

    def position_tokens(self, plan: EncoderPlan) -> Tensor:
        """(b,Nv,C) sine position embedding of the plan's masks in token layout (computed once per plan, on the device,
        by ``self.position_embedding`` -- the detector's module, models/detectors/salience_detr.py:172-176)."""
        pe = getattr(self, "position_embedding", None)
        if pe is None:
            raise RuntimeError("no position embeddings given and no `position_embedding` module attached to the transformer")
        if "pos_tokens" not in plan.scratch:
            plan.scratch["pos_tokens"] = pe.tokens(plan.scratch["ynorm"], plan.scratch["xnorm"])
        return plan.scratch["pos_tokens"]

    # -- salience filter (:112-168) ------------------------------------------------------------------------------
    def salience_filter(self, feat: Tensor, lpos: Tensor, plan: EncoderPlan, want_order: bool = True,
                        x: Optional[Tensor] = None):
        b, nv, c = feat.shape
        L = len(plan.shapes_list)
        # training keeps the scores differentiable (salience supervision): plain torch ops instead of the fused kernels
        grad = torch.is_grad_enabled() and (feat.requires_grad or any(p.requires_grad for p in self.parameters()))
        if x is None:
            x = (feat + lpos) * plan.keep
        if grad:
            mem = self.enc_output_norm(self.enc_output(x))
        else:
            mem = gemm.linear(x, self.enc_output.weight, self.enc_output.bias)
            mem = cabi.add_layernorm(mem, None, self.enc_output_norm.weight, self.enc_output_norm.bias,
                                     self.enc_output_norm.eps, out=mem)
        raw = torch.empty(b, nv, device=feat.device, dtype=torch.float32)
        prev = None
        mp = self.enc_mask_predictor
        small_ok = (not grad and c == 256 and mp.h_dim == 256 and mp.layer1[1].in_features == 256 and
                    mem.is_contiguous())
        for lvl in range(L - 1, -1, -1):
            h, w = plan.shapes_list[lvl]
            s0 = plan.level_start[lvl]
            if small_ok and b * h * w <= PREDICTOR_SMALL_ROWS:  # few rows: launch latency, not arithmetic -- two fused launches
                hc, wc = plan.shapes_list[lvl + 1] if lvl != L - 1 else (0, 0)
                coarse = raw[:, plan.level_start[lvl + 1]:plan.level_start[lvl + 1] + hc * wc] if lvl != L - 1 else None
                ln = mp.layer1[0]
                cabi.mask_predictor_level(mem, s0, h, w, coarse, hc, wc, self.alpha, lvl, ln.weight, ln.bias, ln.eps,
                                          *mp.transposed_weights(), raw, s0)
                continue
            m_l = mem[:, s0:s0 + h * w]
            if lvl != L - 1:
                hc, wc = plan.shapes_list[lvl + 1]
                s1 = plan.level_start[lvl + 1]
                if grad:
                    coarse = prev.transpose(1, 2).reshape(b, 1, hc, wc)
                    if torch.are_deterministic_algorithms_enabled():  # torch's backward of the resize is not deterministic
                        up = UpsampleBilinearAC.apply(coarse, (h, w))
                    else:
                        up = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=True)
                    m_l = m_l + m_l * up.view(b, 1, h * w).transpose(1, 2) * self.alpha[lvl]
                else:
                    m_l = cabi.score_modulate(mem, s0, h, w, raw[:, s1:s1 + hc * wc], hc, wc, self.alpha, lvl)
            prev = self.enc_mask_predictor(m_l) if grad else self.enc_mask_predictor.forward_fast(m_l)
            raw[:, s0:s0 + h * w] = prev.squeeze(-1)
        sel_in = raw.detach() if grad else raw
        inds, score, fg, order = cabi.salience_select(
            sel_in, plan.mask_u8, plan.level_start, plan.level_size, plan.level_token_nums,
            plan.level_width if want_order else None, plan.level_stride if want_order else None, TILE_CELL_PX)
        return raw, inds, score, fg, order

    # -- encoder half ---------------------------------------------------------------------------------------------
    def forward_encoder(self, multi_level_feats, multi_level_masks, multi_level_pos_embeds=None,
                        plan: Optional[EncoderPlan] = None, use_order: bool = True):
        """(b,C,H_l,W_l) feats, (b,H_l,W_l) bool masks, (b,C,H_l,W_l) pos -> memory (b,Nv,C) + aux dict.

        Reference lines 106-183.  Pass a cached ``plan`` (``make_plan``) to run with no host sync.  With gradients enabled (training
        path: torch autograd around the MSDA kernels) the ``nn.Linear`` layers run on the 3xFP16 tensor-core GEMM in forward and
        input-gradient (``gemm.tensor_core_linears``)."""
        grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if grad and multi_level_feats[0].is_cuda:
            with gemm.tensor_core_linears():
                return self._forward_encoder(multi_level_feats, multi_level_masks, multi_level_pos_embeds, plan, use_order)
        return self._forward_encoder(multi_level_feats, multi_level_masks, multi_level_pos_embeds, plan, use_order)

    def _forward_encoder(self, multi_level_feats, multi_level_masks, multi_level_pos_embeds, plan, use_order):
        if plan is None:
            plan = self.make_plan(multi_level_masks)
        grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        x = None
        tokens = None if grad else tokens_of(multi_level_feats)
        if tokens is not None and tokens.is_cuda and tokens.dtype == torch.float32:
            # the features are level views of one token buffer (ChannelMapper): it is the token layout already.  lpos and x are
            # bit-identical to what the flatten kernels make from .contiguous() copies of the same maps
            feat = tokens
            keep, embeds = plan.keep.view(plan.keep.shape[0], -1), self.level_embeds.detach().contiguous()
            if multi_level_pos_embeds is None:
                lpos, x = cabi.token_lpos_keep(feat, self.position_tokens(plan), embeds, keep, plan.level_size)
            else:
                pos = cabi.maps_to_tokens([p.contiguous() for p in multi_level_pos_embeds])
                lpos, x = cabi.token_lpos_keep(feat, pos, embeds, keep, plan.level_size, lpos=pos)
        elif multi_level_pos_embeds is None:  # position embedding computed on the device from the masks, in token layout
            if grad:
                raise RuntimeError("training path: pass the per-level position embeddings explicitly")
            feat, lpos, x = cabi.flatten_tokens_pos([f.contiguous() for f in multi_level_feats], self.position_tokens(plan),
                                                    self.level_embeds.detach().contiguous(), plan.keep.view(plan.keep.shape[0], -1))
        elif grad or multi_level_feats[0].dtype != torch.float32:
            feat = flatten_levels(multi_level_feats)
            lpos = flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(multi_level_pos_embeds, self.level_embeds)])
        else:  # one fused pass: token layout + level embedding + (feat + pos) * keep
            feat, lpos, x = cabi.flatten_tokens([f.contiguous() for f in multi_level_feats],
                                                [p.contiguous() for p in multi_level_pos_embeds],
                                                self.level_embeds.detach().contiguous(), plan.keep.view(plan.keep.shape[0], -1))
        vbuf = None
        if not grad and feat.is_cuda and torch.cuda.is_current_stream_capturing():
            # fork: the (large) value projection only needs the tokens, so it becomes a parallel branch of the captured
            # CUDA graph beside the salience filter's many small kernels.  Not eagerly: there the extra stream operations
            # cost the host-bound path (e.g. the fresh-mask pipeline) more than the overlap returns
            cur = torch.cuda.current_stream(feat.device)
            side = self._side_stream(feat.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                vbuf = self.encoder.project_values(feat, plan.mask_u8)
        raw, inds, score, fg, order = self.salience_filter(feat, lpos, plan, want_order=use_order and not grad, x=x)
        if vbuf is not None:
            cur.wait_stream(side)  # join
            vbuf.record_stream(cur)
        layer_inds = [inds[:, :n] for n in plan.layer_num_query]
        orders = cabi.order_prefixes(order, plan.layer_num_query) if order is not None else None
        memory = self.encoder(
            query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat, spatial_shapes=plan.spatial_shapes,
            level_start_index=plan.level_start_index, valid_ratios=plan.valid_ratios, foreground_score=fg,
            focus_token_nums=plan.focus_token_nums, foreground_inds=layer_inds, multi_level_masks=multi_level_masks,
            query_orders=orders, value_buffer=vbuf, focus_host=plan.focus_host)
        aux = dict(raw_score=raw, selected_inds=inds, selected_score=score, foreground_score=fg, plan=plan)
        return memory, aux

    # -- two-stage proposals (:194-212) ----------------------------------------------------------------------------
    def gen_encoder_output_proposals(self, memory: Tensor, plan: EncoderPlan):
        """base_transformer.py:74-112 on the encoder OUTPUT: (output_memory = LN(Linear(memory * keep)), output_proposals =
        inverse-sigmoid of the (cx, cy, w, h) proposal of every token, +inf where padded / outside (0.01, 0.99))."""
        b, nv, c = memory.shape
        dev = memory.device
        props = []
        for lvl, (h, w) in enumerate(plan.shapes_list):
            vr = plan.valid_ratios[:, lvl]                                  # (b,2) = (valid_w / w, valid_h / h)
            valid_w, valid_h = (vr[:, 0] * w).round(), (vr[:, 1] * h).round()
            gy, gx = torch.meshgrid(torch.linspace(0, h - 1, h, dtype=torch.float32, device=dev),
                                    torch.linspace(0, w - 1, w, dtype=torch.float32, device=dev), indexing="ij")
            grid = torch.stack([gx, gy], -1)
            scale = torch.stack([valid_w, valid_h], -1).view(b, 1, 1, 2)
            grid = (grid.expand(b, -1, -1, -1) + 0.5) / scale
            wh = torch.ones_like(grid) * 0.05 * 2.0 ** lvl
            props.append(torch.cat([grid, wh], -1).view(b, -1, 4))
        output_proposals = torch.cat(props, 1)
        valid = ((output_proposals > 0.01) & (output_proposals < 0.99)).all(-1, keepdim=True)
        output_proposals = torch.log(output_proposals / (1 - output_proposals))
        output_proposals.masked_fill_(plan.mask_flat.unsqueeze(-1) | ~valid, float("inf"))
        grad = torch.is_grad_enabled() and (memory.requires_grad or any(p.requires_grad for p in self.parameters()))
        x = memory * plan.keep  # plan.keep = ~padding & valid, as float (the same predicate, base_transformer.py:100-108)
        if grad:
            output_memory = self.enc_output_norm(self.enc_output(x))
        else:
            y = gemm.linear(x, self.enc_output.weight, self.enc_output.bias)
            output_memory = cabi.add_layernorm(y, None, self.enc_output_norm.weight, self.enc_output_norm.bias,
                                               self.enc_output_norm.eps, out=y)
        return output_memory, output_proposals

    @torch.no_grad()
    def nms_on_topk_index(self, topk_scores, topk_index, spatial_shapes, level_start_index, iou_threshold=0.3,
                          shapes_list=None):
        """Reference :249-295 -> (b, min_num) token indices: NMS of the (x-1, y-1, x+1, y+1) boxes per (image, level) in
        descending score order, first ``two_stage_num_proposals`` survivors, truncated to the batch minimum.  One kernel
        (``sdetr_nms_topk_index``) + the one host read of the survivor counts the reference also needs."""
        shapes = shapes_list if shapes_list is not None else [tuple(int(v) for v in r) for r in spatial_shapes.tolist()]
        kept, count, _ = cabi.nms_topk_index(topk_index.contiguous(), shapes, iou_threshold)
        min_num = min(int(count.min()), self.two_stage_num_proposals)
        return kept[:, :min_num]

    def forward(self, multi_level_feats, multi_level_masks, multi_level_pos_embeds, noised_label_query=None,
                noised_box_query=None, attn_mask=None):
        """Reference call signature and outputs (:97-239): (outputs_classes, outputs_coords, enc_outputs_class,
        enc_outputs_coord, salience_score) when a decoder is attached; (memory, salience maps) for the encoder half alone."""
        memory, aux = self.forward_encoder(multi_level_feats, multi_level_masks, multi_level_pos_embeds)
        plan = aux["plan"]
        b = memory.shape[0]
        salience = [aux["raw_score"][:, s:s + h * w].reshape(b, 1, h, w) for s, (h, w) in zip(plan.level_start, plan.shapes_list)]
        if self.decoder is None and self.neck is None:
            return memory, salience
        if self.neck is not None:  # :185-192 (any nn.Module taking {i: NCHW}; neck.RepVGGPluXNetwork also runs in token layout)
            tokens_ok = getattr(self.neck, "tokens_supported", None)
            training_ok = getattr(self.neck, "training_tokens_supported", None)
            # a training neck takes the token path while a CUDA graph is being captured: replayed it is bound by the device and
            # faster than cuDNN fp32 (tools/bench_neck_train.py); run eagerly its ~1600 launches bind it to the host, where it is
            # no faster than the NCHW route below
            if hasattr(self.neck, "forward_tokens") and (
                    (tokens_ok is not None and tokens_ok(memory, plan.shapes_list)) or
                    (training_ok is not None and torch.cuda.is_current_stream_capturing() and
                     training_ok(memory, plan.shapes_list))):
                memory = self.neck.forward_tokens(memory, plan.shapes_list)
            elif memory.is_cuda and not (torch.is_grad_enabled() and memory.requires_grad):
                feats = dict(enumerate(cabi.tokens_to_maps(memory.contiguous(), plan.shapes_list)))   # one launch each way
                feats = list(self.neck(feats).values())
                memory = cabi.maps_to_tokens([f.float().contiguous() for f in feats])
            else:
                feats = memory.split(plan.level_size, dim=1)
                feats = {i: f.transpose(1, 2).contiguous().reshape(b, self.embed_dim, h, w)
                         for i, (f, (h, w)) in enumerate(zip(feats, plan.shapes_list))}
                feats = list(self.neck(feats).values())
                memory = torch.cat([f.flatten(2).transpose(1, 2) for f in feats], dim=1).contiguous()
            if self.decoder is None:
                return memory, salience
        output_memory, output_proposals = self.gen_encoder_output_proposals(memory, plan)
        grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if grad:
            enc_outputs_class = self.encoder_class_head(output_memory)
        else:
            enc_outputs_class = gemm.linear(output_memory, self.encoder_class_head.weight, self.encoder_class_head.bias)
        enc_outputs_coord = (self.encoder_bbox_head(output_memory) + output_proposals).sigmoid()
        topk = min(self.two_stage_num_proposals * 4, enc_outputs_class.shape[1])
        cls_max = enc_outputs_class.max(-1)[0]
        if cls_max.is_cuda:   # descending score, ties by smaller index (the canonical order of the selection kernels)
            topk_index = cabi.topk_desc(cls_max.detach().float().contiguous(), topk)
            topk_scores = torch.gather(cls_max, 1, topk_index)
        else:
            topk_scores, topk_index = torch.topk(cls_max, topk, dim=1)
        topk_index = self.nms_on_topk_index(topk_scores, topk_index, plan.spatial_shapes, plan.level_start_index, 0.3,
                                            shapes_list=plan.shapes_list).unsqueeze(-1)
        enc_outputs_class = enc_outputs_class.gather(1, topk_index.expand(-1, -1, self.num_classes))
        enc_outputs_coord = enc_outputs_coord.gather(1, topk_index.expand(-1, -1, 4))
        reference_points = enc_outputs_coord.detach()
        target = self.tgt_embed.weight.expand(b, -1, -1)
        if noised_label_query is not None and noised_box_query is not None:
            target = torch.cat([noised_label_query, target], 1)
            reference_points = torch.cat([noised_box_query.sigmoid(), reference_points], 1)
        outputs_classes, outputs_coords = self.decoder(
            query=target, value=memory, key_padding_mask=plan.mask_flat, reference_points=reference_points,
            spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index, valid_ratios=plan.valid_ratios,
            attn_mask=attn_mask)
        return outputs_classes, outputs_coords, enc_outputs_class, enc_outputs_coord, salience
