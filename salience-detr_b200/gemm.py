"""Dense projections of the path (value/output/offset/class projections, FFN, MaskPredictor).

These are true dense GEMMs, the only place of the path where tensor cores belong.  ``MODE``:

* ``"auto"`` (default): the hand-written persistent wgmma kernels on a pre-split weight -- ``OWN_KERNEL = "f16x3"``:
  ``sdetr_gemm_f16x3_pre`` (3xFP16 on ``wgmma`` .f16: same 22-bit operands as 3xTF32 at twice the MMA rate, for
  K % 64 == 0); ``"tf32x3"`` (or K % 64 != 0): ``sdetr_gemm_3xtf32_pre`` -- except GEMMs with at most ``SMALL_M`` rows (the
  coarse levels of the MaskPredictor), which are latency-bound and go to cuBLAS fp32.
* ``"tcgen05"`` (name kept for existing callers): the hand-written sm_90a 3xTF32 GEMM (``sdetr_gemm_3xtf32_pre``: TMA ->
  TF32 split of the activation in registers -> wgmma .tf32 -> epilogue), same arithmetic without the separate split pass.
* ``"3xtf32"``: each operand is split into two TF32 pieces by ``sdetr_split_tf32`` and ONE cuBLAS TF32
  GEMM over K' = 3K accumulates A_hi.B_hi + A_hi.B_lo + A_lo.B_hi in fp32 -- tensor-core speed with fp32-class
  accuracy (error ~2^-21 relative per product, same order as fp32 summation-order noise; measured in
  tests/test_gpu_parity.py::test_linear_3xtf32_accuracy).  Weight splits are cached per parameter version.
* ``"fp32"``: cuBLAS SGEMM on the fp32 SIMT pipe (what the reference runs by default).
* ``"tf32"``: single-pass TF32 (reduced precision; never the bench default).
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional, Tuple

import torch
from torch import Tensor
from torch.nn import functional as F

from . import cabi, derived

MODE = "auto"
OWN_KERNEL = __import__("os").environ.get("SDETR_GEMM_KERNEL", "f16x3")  # "auto" / "tcgen05" own-kernel flavour: "f16x3" (3xFP16, K % 64 == 0) or "tf32x3" (3xTF32)
PRESPLIT_PERSISTENT = True  # persistent kernel fed a pre-split weight (W_hi / W_lo TMA tiles) instead of splitting W in the kernel
LONG_K_PRESPLIT = False  # K >= 1024: True = "SS" kernel with the pre-split weight, False = persistent raw-weight kernel "P" (measured equal or faster)
SMALL_M = 2304  # "auto": at most this many rows -> cuBLAS fp32 (latency-bound; measured faster than either tensor-core path, tools/bench_small.py)
K_CHUNK = 512  # longest reduction handed to one tensor-core GEMM (its accumulator truncates: error ~ length)


@contextlib.contextmanager
def _tf32_matmul():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def _chunk_of(K: int) -> int:
    return K_CHUNK if K > K_CHUNK and K % K_CHUNK == 0 else K


def split_weight(weight: Tensor) -> Tensor:
    """(N,K) -> cached (N,3K) per-chunk [hi|lo|hi]; rebuilt when the parameter is modified in place or replaced."""
    return derived.cached(weight, "split_tf32", (weight,), lambda: cabi.split_tf32(
        weight.detach().contiguous(), layout_b=True, chunk=_chunk_of(weight.shape[1])))


def split_weight_pair(weight: Tensor) -> Tuple[Tensor, Tensor]:
    return derived.cached(weight, "split_tf32_pair", (weight,), lambda: cabi.split_tf32_pair(weight.detach()))


def split_weight_f16(weight: Tensor):
    """(N,K) -> cached (W_hi fp16, W_lo fp16, power-of-two scale); one host read of max|W| per parameter version."""
    return derived.cached(weight, "split_f16_pair", (weight,), lambda: cabi.split_f16_pair(weight.detach()))


_ACT = {None: 0, "relu": 1, "gelu": 2}


def _act_torch(x: Tensor, act) -> Tensor:
    return F.relu(x) if act == 1 else F.gelu(x) if act == 2 else x


def _native(x: Tensor, weight: Tensor, bias: Optional[Tensor]) -> bool:
    """Operands the project's kernels take: fp32 CUDA tensors on the current device (any layout), a 2-D weight, at least
    one row.  Everything else F.linear accepts (other dtypes, CPU tensors, empty inputs) goes to F.linear."""
    return (x.is_cuda and weight.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32 and
            weight.dim() == 2 and x.numel() > 0 and x.device == weight.device and x.device.index == cabi._current_device()
            and (bias is None or (bias.is_cuda and bias.dtype == torch.float32 and bias.device == x.device)))


def _rows(x: Tensor) -> Tensor:
    """x (..., K) as the (rows, K) operand the kernels read in place -- unit last stride, one row pitch that is a multiple
    of 4 floats, a 16-byte aligned base -- or, for any other layout F.linear accepts (transposed, odd pitch, an offset
    view, non-uniform batch strides), an aligned contiguous copy of it."""
    x2 = x if x.dim() == 2 else x.reshape(-1, x.shape[-1])  # a fresh contiguous copy when the rows are not uniformly strided
    if x2.data_ptr() != x.data_ptr() or (x2.stride(-1) == 1 and (x2.stride(0) % 4 == 0 or x2.shape[0] == 1) and
                                         x2.data_ptr() % 16 == 0):
        return x2
    return x2.clone(memory_format=torch.contiguous_format)


def f16x3_route(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None) -> bool:
    """True when ``linear(x, weight, bias)`` (no input activation) runs ``sdetr_gemm_f16x3_pre``.  The kernels that fuse a
    consumer into that GEMM's epilogue (``cabi.gemm_f16x3_rowmax``, ``cabi.gemm_f16x3_add_layernorm_``) reproduce its product
    bit for bit, so callers take them exactly where ``linear`` would have taken this route."""
    k = weight.shape[-1]
    return (MODE == "auto" and OWN_KERNEL == "f16x3" and k % 64 == 0 and not (k >= 1024 and LONG_K_PRESPLIT) and
            x.numel() // max(k, 1) > SMALL_M and _native(x, weight, bias))


def linear(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None, relu_input: bool = False,
           input_act: Optional[str] = None) -> Tensor:
    """y = act(x) @ weight.T + bias (act: None | "relu" | "gelu", fused into the operand load / split), inference only.
    A drop-in for F.linear: any input it accepts works (see ``_native`` and ``_rows``)."""
    relu_input = 1 if relu_input else _ACT[input_act]
    n, k = weight.shape[0], weight.shape[-1]
    if (MODE == "auto" and x.numel() // max(k, 1) <= SMALL_M) or not _native(x, weight, bias):
        return F.linear(_act_torch(x, relu_input), weight, bias)
    bias = bias if bias is None or bias.is_contiguous() else bias.contiguous()
    own = MODE in ("tcgen05", "auto")
    if own and k % 32 == 0:
        x2 = _rows(x)
        if k >= 1024 and LONG_K_PRESPLIT:   # long reductions: 4-stage ring, weight pre-split once (variant "SS")
            w_hi, w_lo = split_weight_pair(weight)
            y = cabi.gemm_3xtf32(x2, w_hi, w_lo, bias, relu_input)
        elif OWN_KERNEL == "f16x3" and MODE == "auto" and k % 64 == 0:
            w_hi, w_lo, w_scale = split_weight_f16(weight)
            y = cabi.gemm_f16x3_pre(x2, w_hi, w_lo, w_scale, bias, relu_input)
        elif PRESPLIT_PERSISTENT:
            w_hi, w_lo = split_weight_pair(weight)
            y = cabi.gemm_3xtf32_pre(x2, w_hi, w_lo, bias, relu_input)
        else:  # both operands split in the kernel
            y = cabi.gemm_3xtf32_raw(x2, weight if weight.is_contiguous() else weight.contiguous(), bias, relu_input)
        return y.reshape(*x.shape[:-1], n)
    if MODE == "fp32" or k % 4 != 0:
        return F.linear(_act_torch(x, relu_input), weight, bias)
    if MODE == "tf32":
        with _tf32_matmul():
            return F.linear(_act_torch(x, relu_input), weight, bias)
    K = weight.shape[1]
    kc = _chunk_of(K)  # (MODE "3xtf32", or "tcgen05" falling back for an unsupported shape)
    x3 = cabi.split_tf32(_rows(x), layout_b=False, relu=relu_input, chunk=kc)
    w3 = split_weight(weight)
    with _tf32_matmul():
        if kc == K:
            y = F.linear(x3, w3, bias)
        else:  # long reduction: one GEMM per K-chunk, accumulated in fp32 by the epilogue (beta = 1)
            y = F.linear(x3[:, :3 * kc], w3[:, :3 * kc], bias)
            for c in range(1, K // kc):
                y.addmm_(x3[:, 3 * kc * c:3 * kc * (c + 1)], w3[:, 3 * kc * c:3 * kc * (c + 1)].t())
    return y.view(*x.shape[:-1], weight.shape[0])


# ---- training path: tensor-core Linear with autograd ---------------------------------------------------------------------------
TRAIN_TENSOR_CORE = __import__("os").environ.get("SDETR_TRAIN_TENSOR_CORE", "1") != "0"
_const16: Dict[int, Tensor] = {}


def _split_train(weight: Tensor):
    w = weight.detach()
    scale = cabi.pow2_scale(w if w.is_contiguous() else w.contiguous(), 14)
    fwd = cabi.split_f16_pair_dev(w, scale)
    bwd = cabi.split_f16_pair_dev(w.t().contiguous(), scale) if w.shape[0] % 64 == 0 else None
    return fwd, bwd


def _train_splits(weight: Tensor):
    """Per parameter VERSION (the optimizer bumps it every step): device-side power-of-two scale, the 3xFP16 split of W (for y)
    and of W^T (for dx).  Everything stays on the device -- no host read of max|W|, unlike ``split_weight_f16``."""
    # inside a CUDA-graph capture of a training step the split kernels must be PART of the graph (the optimizer rewrites the
    # weights on every replay, and no Python runs then): never serve a capture from the cache, never cache what it produced
    if weight.is_cuda and torch.cuda.is_current_stream_capturing():
        return _split_train(weight)
    return derived.cached(weight, "train_splits", (weight,), lambda: _split_train(weight))


class _LinearF16x3(torch.autograd.Function):
    """y = x W^T + b on the 3xFP16 tensor-core kernel, forward AND the input gradient (dx = dy W: the same kernel on W^T, with dy
    scaled by a device-side power of two -- gradients are far below the fixed activation range of the inference entry point);
    dW = dy^T x stays on cuBLAS fp32 (a K = rows reduction into a small output: split-K territory, which the persistent kernel
    does not do)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        (w_hi, w_lo, w_scale), ctx.bwd = _train_splits(weight)   # the W^T split rides along for the input gradient
        c16 = _const16.get(x.device.index)
        if c16 is None:
            c16 = _const16[x.device.index] = torch.full((1,), 16.0, device=x.device)
        y = cabi.gemm_f16x3_scaled(_rows(x).view(x.shape), c16, w_hi, w_lo, w_scale, bias)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not (dy2.is_contiguous() and dy2.data_ptr() % 16 == 0):  # pow2_scale and the kernel read it as one aligned block
            dy2 = dy2.clone(memory_format=torch.contiguous_format)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            bwd = ctx.bwd
            if bwd is not None:
                dx = cabi.gemm_f16x3_scaled(dy2, cabi.pow2_scale(dy2, 12), bwd[0], bwd[1], bwd[2]).reshape(x.shape)
            else:
                dx = (dy2 @ weight).reshape(x.shape)
        if ctx.needs_input_grad[1]:
            dw = dy2.t() @ x.reshape(-1, x.shape[-1])
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.sum(0)
        return dx, dw, db


def linear_train(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None) -> Tensor:
    """Differentiable ``F.linear`` for the training path: tensor cores where the shapes allow (K % 64 == 0, more than SMALL_M
    rows, fp32 CUDA on the current device, any layout), ``F.linear`` otherwise."""
    rows = x.numel() // max(x.shape[-1], 1)
    if (TRAIN_TENSOR_CORE and MODE == "auto" and OWN_KERNEL == "f16x3" and _native(x, weight, bias) and
            x.shape[-1] % 64 == 0 and rows > SMALL_M):
        return _LinearF16x3.apply(x, weight, bias if bias is None or bias.is_contiguous() else bias.contiguous())
    return _orig_linear(x, weight, bias)


_orig_linear = F.linear


@contextlib.contextmanager
def tensor_core_linears():
    """Inside: every ``torch.nn.functional.linear`` (``nn.Linear.forward``, ``nn.MultiheadAttention``) of the training path goes
    through ``linear_train``.  Used by ``SalienceTransformer.forward_encoder`` when gradients are enabled."""
    if not TRAIN_TENSOR_CORE:
        yield
        return
    prev = torch.nn.functional.linear
    torch.nn.functional.linear = linear_train
    try:
        yield
    finally:
        torch.nn.functional.linear = prev
