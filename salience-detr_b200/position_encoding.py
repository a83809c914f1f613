"""Drop-in mirror of the reference's ``PositionEmbeddingSine`` (models/bricks/position_encoding.py:9-65).

Same constructor arguments and buffers (``dim_tx`` / ``dim_ty``) and the same ``forward(mask) -> (b, 2F, H, W)``.
In the detector the embedding is a pure function of the padding mask (models/detectors/salience_detr.py:172-176), so the
H100 path never moves it over PCIe and never materialises it per level in NCHW: ``tokens()`` writes it once per mask
geometry, directly in the (b,Nv,C) token layout the encoder consumes, from the normalised coordinates that
``sdetr_mask_plan`` produces (two launches instead of ~15 ATen launches per level)."""
from __future__ import annotations

import math
from typing import Tuple, Union

import torch
from torch import Tensor, nn

from . import cabi


class PositionEmbeddingSine(nn.Module):
    def __init__(self, num_pos_feats=64, temperature: Union[int, Tuple[int, int]] = 10000, normalize=False,
                 scale=2 * math.pi, eps=1e-6, offset=0.0):
        super().__init__()
        dim_t = 2 * torch.arange(num_pos_feats).div(2, rounding_mode="floor") / num_pos_feats
        if isinstance(temperature, int):
            dim_tx = dim_ty = temperature ** dim_t
        else:
            assert len(temperature) == 2, "Only support two elements as (t_x, t_y) in temperature"
            dim_tx, dim_ty = [t ** dim_t for t in temperature]
        self.register_buffer("dim_tx", dim_tx)
        self.register_buffer("dim_ty", dim_ty)
        self.num_pos_feats = num_pos_feats
        self.normalize, self.scale, self.eps, self.offset = normalize, scale, eps, offset

    def tokens(self, ynorm: Tensor, xnorm: Tensor) -> Tensor:
        """(b,Nv) normalised coordinates (``cabi.mask_plan``) -> (b,Nv,2F) embedding in token layout."""
        if not self.normalize:
            raise RuntimeError("the fused token path implements normalize=True (every Salience-DETR config)")
        dev = ynorm.device
        if self.__dict__.get("_dev_tables", (None,))[0] != dev:  # the module may live outside a model's .to(device)
            self.__dict__["_dev_tables"] = (dev, self.dim_ty.to(dev, torch.float32).contiguous(),
                                            self.dim_tx.to(dev, torch.float32).contiguous())
        _, ty, tx = self.__dict__["_dev_tables"]
        return cabi.sine_pos_tokens(ynorm, xnorm, ty, tx)

    def forward(self, mask: Tensor) -> Tensor:
        """Reference signature: (b,H,W) bool padding mask -> (b,2F,H,W).  CUDA masks run the fused kernels."""
        if not mask.is_cuda:
            raise RuntimeError("PositionEmbeddingSine needs a CUDA mask; there is no CPU path")
        b, h, w = mask.shape
        if not self.normalize:  # RT-DETR style un-normalised variant: not on this path, plain torch ops
            nm = (~mask.bool()).to(torch.float32)
            y, x = nm.cumsum(1) + self.offset, nm.cumsum(2) + self.offset
            px, py = x[..., None] / self.dim_tx, y[..., None] / self.dim_ty
            px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=4).flatten(3)
            py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=4).flatten(3)
            return torch.cat((py, px), dim=3).permute(0, 3, 1, 2)
        plan = cabi.mask_plan(mask.reshape(b, h * w).to(torch.uint8).contiguous(), [(h, w)], [1.0], self.offset, self.eps,
                              self.scale)
        return self.tokens(plan["ynorm"], plan["xnorm"]).view(b, h, w, -1).permute(0, 3, 1, 2)
