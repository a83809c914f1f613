"""Drop-in mirror of the reference's ``models/bricks/ms_deform_attn.py`` on top of the sm_90a C-ABI.

Same public names, constructor arguments, parameter names and ``forward`` signature as the reference
(``MultiScaleDeformableAttention`` ms_deform_attn.py:215-377, ``MultiScaleDeformableAttnFunction`` :35-84,
the ``_C`` operator pair ms_deform_attn_cuda.cu:148-151), so reference configs and checkpoints load
unchanged.  Differences are all behind the boundary:

* the core always runs the hand-written kernel (``cabi``); there is no PyTorch ``grid_sample`` fallback
  and no JIT build at import time (the reference's extension does not compile against torch 2.11 and
  silently falls back, ms_deform_attn.py:14-26);
* in inference (no grad) the attention softmax, the sampling-location arithmetic and the sampling are
  ONE fused launch fed by one concatenated ``sampling_offsets|attention_weights`` GEMM;
* no host synchronisation (the reference asserts on a device reduction, :313).
"""
from __future__ import annotations

import math
import warnings
from types import SimpleNamespace
from typing import Optional

import torch
from torch import Tensor, nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn import functional as F

from . import cabi, gemm


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step=64):
    """Operator-level replacement of ``_C.ms_deform_attn_forward`` (ms_deform_attn_cuda.cu:12-72).

    ``im2col_step`` is accepted for signature compatibility; the reference only uses it to chunk the batch
    (no numerical effect), and enforces ``batch % min(batch, im2col_step) == 0`` (.cu:42-44)."""
    step = min(value.shape[0], im2col_step)
    if value.shape[0] % step != 0:
        raise RuntimeError(f"batch({value.shape[0]}) must divide im2col_step({step})")
    return cabi.msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight)


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                            im2col_step=64):
    """Operator-level replacement of ``_C.ms_deform_attn_backward`` (ms_deform_attn_cuda.cu:75-145)."""
    step = min(value.shape[0], im2col_step)
    if value.shape[0] % step != 0:
        raise RuntimeError(f"batch({value.shape[0]}) must divide im2col_step({step})")
    return list(cabi.msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output))


# what `from models.bricks.ms_deform_attn import _C` gives the reference code
_C = SimpleNamespace(ms_deform_attn_forward=ms_deform_attn_forward, ms_deform_attn_backward=ms_deform_attn_backward)


class MultiScaleDeformableAttnFunction(Function):
    """Same six inputs / three gradients as the reference Function (ms_deform_attn.py:35-84)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        ctx.im2col_step = im2col_step
        out = ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                                     attention_weights, im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                              attention_weights)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, lsi, loc, attn = ctx.saved_tensors
        gv, gl, ga = ms_deform_attn_backward(value, shapes, lsi, loc, attn, grad_output.contiguous(), ctx.im2col_step)
        return gv, None, None, gl, ga, None


class MultiScaleDeformableAttention(nn.Module):
    """Multi-scale deformable attention (Deformable-DETR), H100-native core."""

    def __init__(self, embed_dim: int = 256, num_levels: int = 4, num_heads: int = 8, num_points: int = 4,
                 img2col_step: int = 64):
        super().__init__()
        if embed_dim % num_heads != 0:
            raise ValueError(f"embed_dim must be divisible by num_heads, but got {embed_dim} and {num_heads}")
        head_dim = embed_dim // num_heads
        if head_dim & (head_dim - 1):
            warnings.warn("embed_dim / num_heads should be a power of 2 for the 128-bit row kernels")
        self.im2col_step = img2col_step
        self.embed_dim, self.num_heads, self.num_levels, self.num_points = embed_dim, num_heads, num_levels, num_points
        n = num_heads * num_levels * num_points
        self.sampling_offsets = nn.Linear(embed_dim, 2 * n)
        self.attention_weights = nn.Linear(embed_dim, n)
        self.value_proj = nn.Linear(embed_dim, embed_dim)
        self.output_proj = nn.Linear(embed_dim, embed_dim)
        self._fused_w: Optional[Tensor] = None
        self._fused_b: Optional[Tensor] = None
        self._fused_key = None
        self.init_weights()

    def init_weights(self):
        """Reference initialisation (ms_deform_attn.py:266-284): zero offset weights, offset bias = ring of
        num_heads directions scaled by the point index, zero attention weights, Xavier projections."""
        M, L, P = self.num_heads, self.num_levels, self.num_points
        ang = torch.arange(M, dtype=torch.float32) * (2.0 * math.pi / M)
        ring = torch.stack([ang.cos(), ang.sin()], -1)
        ring = ring / ring.abs().max(-1, keepdim=True)[0]
        bias = ring.view(M, 1, 1, 2).repeat(1, L, P, 1) * torch.arange(1, P + 1, dtype=torch.float32).view(1, 1, P, 1)
        with torch.no_grad():
            self.sampling_offsets.weight.zero_()
            self.sampling_offsets.bias.copy_(bias.reshape(-1))
            self.attention_weights.weight.zero_()
            self.attention_weights.bias.zero_()
            nn.init.xavier_uniform_(self.value_proj.weight)
            self.value_proj.bias.zero_()
            nn.init.xavier_uniform_(self.output_proj.weight)
            self.output_proj.bias.zero_()
        self._fused_w = None

    # -- inference fast path --------------------------------------------------------------------------------
    def fused_projection(self):
        """Concatenated [sampling_offsets | attention_weights] weight/bias (one GEMM, N = 3*M*L*P)."""
        so, aw = self.sampling_offsets, self.attention_weights
        key = (so.weight.data_ptr(), so.weight._version, so.bias._version, aw.weight._version, aw.bias._version)
        if self._fused_w is None or self._fused_key != key:  # rebuilt after load_state_dict / optimizer steps
            self._fused_key = key
            with torch.no_grad():
                self._fused_w = torch.cat([self.sampling_offsets.weight, self.attention_weights.weight], 0).contiguous()
                self._fused_b = torch.cat([self.sampling_offsets.bias, self.attention_weights.bias], 0).contiguous()
        return self._fused_w, self._fused_b

    def project_value(self, value: Tensor, key_padding_mask: Optional[Tensor]) -> Tensor:
        """value_proj + zeroing of padded rows (ms_deform_attn.py:316-321) -> (b,Nv,M,D)."""
        b, nv, _ = value.shape
        train = torch.is_grad_enabled() and (value.requires_grad or self.value_proj.weight.requires_grad)
        v = self.value_proj(value) if train else gemm.linear(value, self.value_proj.weight, self.value_proj.bias)
        if key_padding_mask is not None:
            if train:
                v = v.masked_fill(key_padding_mask[..., None], 0.0)
            else:
                cabi.zero_masked_rows_(v, self.embed_dim, self.embed_dim, key_padding_mask.to(torch.uint8).contiguous(),
                                       b * nv)
        return v.view(b, nv, self.num_heads, self.embed_dim // self.num_heads)

    def forward_projected(self, query: Tensor, reference_points: Tensor, value_buf: Tensor, value_batch_stride: int,
                          value_token_stride: int, value_offset: int, num_value: int, spatial_shapes: Tensor,
                          level_start_index: Tensor, query_order: Optional[Tensor] = None, schedule: int = 0,
                          value_ready=None, proj: Optional[Tensor] = None) -> Tensor:
        """Inference path with an already projected (and masked) value buffer; 2-d reference points.  ``value_ready``:
        optional callable run right before the sampling launch (joins the stream that produces ``value_buf``)."""
        if proj is None:  # else: the caller computed the offsets|logits projection already (overlapped with other work)
            w, b = self.fused_projection()
            proj = gemm.linear(query, w, b)
        if value_ready is not None:
            value_buf = value_ready()
        out = cabi.msda_fused_forward(value_buf, value_batch_stride, value_token_stride, value_offset, spatial_shapes,
                                      level_start_index, reference_points, proj, self.num_heads,
                                      self.embed_dim // self.num_heads, self.num_levels, self.num_points, num_value,
                                      query_order, schedule)
        return gemm.linear(out, self.output_proj.weight, self.output_proj.bias)

    def forward(self, query: Tensor, reference_points: Tensor, value: Tensor, spatial_shapes: Tensor,
                level_start_index: Tensor, key_padding_mask: Tensor) -> Tensor:
        """Same contract as the reference forward (ms_deform_attn.py:286-377).

        query (b,Nq,C); reference_points (b,Nq,L,2) or (b,Nq,L,4); value (b,Nv,C); spatial_shapes (L,2) int64;
        level_start_index (L,) int64; key_padding_mask (b,Nv) bool or None -> (b,Nq,C)."""
        b, nq, _ = query.shape
        nv = value.shape[1]
        if not value.is_cuda:
            raise RuntimeError("MultiScaleDeformableAttention needs CUDA tensors; there is no CPU path")
        M, L, P, D = self.num_heads, self.num_levels, self.num_points, self.embed_dim // self.num_heads
        v = self.project_value(value, key_padding_mask)
        needs_grad = torch.is_grad_enabled() and (query.requires_grad or v.requires_grad or
                                                  any(p.requires_grad for p in self.parameters()))
        if reference_points.shape[-1] == 2 and not needs_grad:
            v32 = v if v.dtype == torch.float32 else v.float()
            out = self.forward_projected(query.float(), reference_points.float().contiguous(), v32, nv * M * D, M * D,
                                         0, nv, spatial_shapes, level_start_index)
            return out.to(value.dtype) if value.dtype != torch.float32 else out
        off = self.sampling_offsets(query).view(b, nq, M, L, P, 2)
        attn = self.attention_weights(query).view(b, nq, M, L * P).softmax(-1).view(b, nq, M, L, P)
        if reference_points.shape[-1] == 2:
            norm = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
            loc = reference_points[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
        elif reference_points.shape[-1] == 4:  # reference boxes (decoder), ms_deform_attn.py:345-349
            loc = reference_points[:, :, None, :, None, :2] + off / P * reference_points[:, :, None, :, None, 2:] * 0.5
        else:
            raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {reference_points.shape[-1]} instead.")
        out = MultiScaleDeformableAttnFunction.apply(v.to(torch.float32).contiguous(), spatial_shapes, level_start_index,
                                                     loc.float().contiguous(), attn.float().contiguous(),
                                                     self.im2col_step)
        if v.dtype != torch.float32:
            out = out.to(v.dtype)
        return self.output_proj(out)
