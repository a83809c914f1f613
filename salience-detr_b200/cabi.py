"""ctypes binding of the C-ABI library declared in ``include/sdetr_b200.h``.

PyTorch is plumbing only here: it owns device memory and the stream; every wrapper validates its
tensors the way the reference op does (contiguous + CUDA, ``AT_ASSERTM`` in
models/bricks/ops/cuda/ms_deform_attn_cuda.cu:20-30), allocates the outputs with ``torch.empty`` and passes
raw pointers plus ``torch.cuda.current_stream().cuda_stream``.  A non-zero return code becomes a
``RuntimeError`` carrying ``sdetr_last_error()``.

There is NO fallback: if the shared library is missing the import of the product path fails loudly.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsdetr_b200.so")
_lib = None

_vp, _i, _i64, _sz, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_size_t, ctypes.c_float

# name -> (restype, argtypes); must list every symbol of include/sdetr_b200.h (tests check this)
SIGNATURES = {
    "sdetr_version": (_i, []),
    "sdetr_last_error": (ctypes.c_char_p, []),
    "sdetr_launch_count": (ctypes.c_ulonglong, []),
    "sdetr_set_persistent_ctas": (_i, [_i]),
    "sdetr_set_option": (_i, [ctypes.c_char_p, _i]),
    "sdetr_msda_forward": (_i, [_vp] * 6 + [_i] * 7 + [_vp]),
    "sdetr_msda_forward_ex": (_i, [_vp, _i64, _i64] + [_vp] * 5 + [_i] * 7 + [_vp, _i, _vp]),
    "sdetr_msda_fused_forward": (_i, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp] + [_i] * 7 + [_vp, _i, _vp]),
    "sdetr_msda_fused_forward_boxes": (_i, [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp] + [_i] * 7 + [_vp, _i, _vp]),
    "sdetr_msda_set_host_shapes": (_i, [_i, _vp, _vp]),
    "sdetr_nms_topk_index": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp]),
    "sdetr_msda_backward": (_i, [_vp] * 9 + [_i] * 7 + [_vp]),
    "sdetr_msda_backward_deterministic_workspace": (_sz, [_i] * 4),
    "sdetr_msda_backward_deterministic": (_i, [_vp] * 9 + [_i] * 7 + [_vp, _sz, _vp]),
    "sdetr_upsample_bilinear_ac_backward": (_i, [_vp] + [_i] * 5 + [_vp, _vp]),
    "sdetr_salience_select_workspace": (_sz, [_i, _i, _i]),
    "sdetr_salience_select": (_i, [_vp] * 7 + [_i] * 4 + [_vp] * 5 + [_sz, _vp]),
    "sdetr_order_prefixes": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "sdetr_topk_workspace": (_sz, [_i, _i]),
    "sdetr_topk_desc": (_i, [_vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "sdetr_token_gather": (_i, [_vp] * 5 + [_i64, _vp, _vp] + [_i] * 5 + [_vp] * 6),
    "sdetr_token_scatter": (_i, [_vp, _vp, _vp, _i64, _vp] + [_i] * 4 + [_vp]),
    "sdetr_background_embed": (_i, [_vp, _vp, _vp, _i64, _i, _vp, _vp, _i, _vp, _vp, _vp] + [_i] * 4 + [_vp, _vp]),
    "sdetr_score_modulate": (_i, [_vp, _i64, _vp, _i64, _vp] + [_i] * 7 + [_vp, _vp]),
    "sdetr_zero_masked_rows": (_i, [_vp, _i64, _i, _vp, _i64, _vp]),
    "sdetr_gelu_colmean_workspace": (_sz, [_i, _i, _i, _i]),
    "sdetr_gelu_colmean": (_i, [_vp, _i, _i, _i, _i, _vp, _sz, _vp]),
    "sdetr_class_max_times_fg": (_i, [_vp, _i64, _vp, _i64, _i, _vp, _vp]),
    "sdetr_add_layernorm": (_i, [_vp, _vp, _vp, _vp, _f, _i64, _i, _vp, _vp]),
    "sdetr_split_tf32": (_i, [_vp, _i64, _i64, _i, _i, _i, _i, _vp, _vp]),
    "sdetr_gemm_3xtf32_raw": (_i, [_vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp]),
    "sdetr_split_tf32_pair": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "sdetr_gemm_3xtf32": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp]),
    "sdetr_gemm_3xtf32_pre": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _vp]),
    "sdetr_flatten_tokens_pos": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "sdetr_salience_targets": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sdetr_token_map_transpose": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "sdetr_mask_plan": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sdetr_sine_pos_tokens": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _vp, _vp]),
    "sdetr_split_f16_pair": (_i, [_vp, _i64, _f, _vp, _vp, _vp]),
    "sdetr_gemm_f16x3_pre": (_i, [_vp, _i64, _vp, _vp, _f, _vp, _vp, _i64, _i, _i, _i, _i, _vp]),
    "sdetr_gemm_f16x3_scaled": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp]),
    "sdetr_split_f16_pair_dev": (_i, [_vp, _i64, _vp, _vp, _vp, _vp]),
    "sdetr_pow2_scale": (_i, [_vp, _i64, _i, _vp, _vp, _vp]),
    "sdetr_mask_predictor_level_workspace_floats": (_i64, [_i, _i, _i]),
    "sdetr_mask_predictor_level": (_i, [_vp, _i64, _i, _i, _i, _i, _vp, _i64, _i, _i, _vp, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _i64, _vp, _i64, _vp]),
    "sdetr_gemm_f16x3_rowmax": (_i, [_vp, _i64, _vp, _vp, _f, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "sdetr_gemm_f16x3_add_layernorm": (_i, [_vp, _i64, _vp, _vp, _f, _vp, _vp, _vp, _f, _vp, _i, _vp]),
    "sdetr_ffn_fused_workspace_floats": (_i64, [_i, _i]),
    "sdetr_ffn_fused_layernorm": (_i, [_vp, _i64, _vp, _vp, _f, _vp, _vp, _vp, _f, _vp, _vp, _vp, _f, _i, _i, _vp, _i64, _vp, _vp]),
    "sdetr_flatten_set_vectorized": (_i, [_i]),
    "sdetr_flatten_tokens": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "sdetr_attention_qkv": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "sdetr_mha_in_proj": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "sdetr_mha_out_proj_ln_scatter": (_i, [_vp] * 6 + [_f, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "sdetr_rows_gather_add": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "sdetr_rows_scatter": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "sdetr_conv2d_f16x3": (_i, [_vp, _i64, _i64, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i, _i, _i, _i, _i,
                                _vp, _i64, _i64, _vp]),
    "sdetr_context_gate_workspace_floats": (_i64, [_i, _i, _i]),
    "sdetr_context_gate": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp, _i64, _i64, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i64, _vp,
                                _i64, _i64, _vp]),
    "sdetr_upsample_nearest_concat": (_i, [_vp, _i64, _i64, _i, _i, _vp, _i64, _i64, _i, _i, _i, _i, _vp, _i64, _i64, _vp]),
    "sdetr_conv2d_f16x3_split_weight": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sdetr_conv2d_f16x3_wgrad_workspace_floats": (_i64, [_i] * 7),
    "sdetr_conv2d_f16x3_wgrad": (_i, [_vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp] + [_i] * 8 + [_vp, _vp, _i64, _vp, _vp]),
    "sdetr_upsample_nearest_concat_backward": (_i, [_vp, _i64, _i64, _i, _i, _i, _i, _i, _i, _vp, _i64, _i64, _vp]),
    "sdetr_group_norm_tokens_workspace_floats": (_i64, [_i, _i, _i, _i, _vp]),
    "sdetr_group_norm_tokens": (_i, [_vp, _vp, _i64, _i, _i, _i, _vp, _vp, _vp, _i, _f, _vp, _i64, _vp]),
    "sdetr_group_norm_tokens_backward_workspace_floats": (_i64, [_i, _i, _i, _i, _vp]),
    "sdetr_group_norm_tokens_backward": (_i, [_vp, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _i, _f, _vp, _vp, _vp, _i64, _vp]),
    "sdetr_token_lpos_keep": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "sdetr_set_match_workspace_floats": (_i64, [_vp, _i]),
    "sdetr_set_match": (_i, [_vp, _i, _i, _f, _f, _f, _f, _f, _vp, _vp, _i64, _vp]),
    "sdetr_set_assign": (_i, [_vp, _i, _vp, _i64, _vp, _vp]),
    "sdetr_set_loss_workspace_floats": (_i64, [_vp, _i]),
    "sdetr_set_loss_forward": (_i, [_vp, _i, _i, _i, _f, _f, _vp, _f, _vp, _vp, _i64, _vp, _vp]),
    "sdetr_set_loss_backward": (_i, [_vp, _i, _i, _i, _f, _f, _vp, _f, _vp, _vp, _vp]),
    "sdetr_cdn_queries": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp] + [_i] * 7 + [_vp] * 6),
    "sdetr_cdn_queries_backward": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "sdetr_cdn_loss_indices": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "sdetr_postprocess_workspace": (_sz, [_i, _i, _i]),
    "sdetr_postprocess": (_i, [_vp, _i64, _i64, _vp, _i64, _i64, _vp] + [_i] * 5 + [_f, _f] + [_vp] * 5 + [_sz, _vp]),
    "sdetr_resnet_stem": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "sdetr_maxpool3x3s2_tokens": (_i, [_vp, _i64, _i64, _i, _i, _i, _i, _vp, _i64, _i64, _vp]),
    "sdetr_conv2d_f16x3_dgrad": (_i, [_vp, _i64, _i64, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i64, _i64] + [_i] * 6 +
                                 [_vp, _i64, _i64, _vp]),
    "sdetr_frozen_bn_fold": (_i, [_vp, _i, _i64, _vp, _vp, _vp, _vp, ctypes.c_double, _vp, _vp, _vp, _vp]),
    "sdetr_gemm_f16x3_ex": (_i, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _vp]),
    "sdetr_convnext_stem": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    "sdetr_dwconv7x7_layernorm_tokens": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    "sdetr_layernorm_tokens_s2d": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _vp, _vp]),
    "sdetr_window_attention_tokens": (_i, [_vp, _vp, _vp] + [_i] * 9 + [_vp, _vp]),
    "sdetr_patch_merge_layernorm_tokens": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _f, _vp, _vp]),
    "sdetr_layernorm_tokens": (_i, [_vp, _i64, _i, _vp, _vp, _f, _vp, _vp]),
    "sdetr_focalnet_stem": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _vp, _vp]),
    "sdetr_focal_context_workspace_floats": (_i64, [_i, _i, _i, _i]),
    "sdetr_focal_level_tokens": (_i, [_vp, _i64, _vp, _i64, _vp] + [_i] * 6 + [_vp, _vp, _vp, _i64, _vp]),
    "sdetr_focal_global_context": (_i, [_vp, _i64, _vp, _i64] + [_i] * 6 + [_vp, _vp]),
    "sdetr_focal_modulate": (_i, [_vp, _i64, _vp, _i64, _i, _vp, _vp]),
    "sdetr_layernorm_scale_add_tokens": (_i, [_vp, _i64, _i, _vp, _vp, _f, _vp, _vp, _vp]),
}


def lib():
    """Load (once) the sm_90a library.  Raises if it has not been built (``__graft_entry__.build()``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). There is no CPU or PyTorch fallback for this path.")
        cdll = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(cdll, name)
            fn.restype, fn.argtypes = res, args
        _lib = cdll
    return _lib


def set_option(name: str, value: int):
    _check(lib().sdetr_set_option(name.encode(), int(value)), "sdetr_set_option")


def launch_count() -> int:
    return int(lib().sdetr_launch_count())


def _check(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"{what} failed (rc={rc}): {lib().sdetr_last_error().decode()}")


# The eager path issues ~120 launches per forward from Python; `torch.cuda.current_stream()` / `current_device()` cost several
# microseconds each (device-index resolution, Stream object construction) and were a third of the host time per forward
# (tools/profile_eager_cpu.py).  The raw accessors below return the same values.
_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_raw_device = getattr(torch._C, "_cuda_getDevice", None)


def _stream() -> int:
    if _raw_stream is not None and _raw_device is not None:
        return _raw_stream(_raw_device())
    return torch.cuda.current_stream().cuda_stream


def _current_device() -> int:
    return _raw_device() if _raw_device is not None else torch.cuda.current_device()


def _req(t: torch.Tensor, name: str, dtype=None):
    # same contract as the reference's AT_ASSERTM checks -> RuntimeError
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.device.index != _current_device():
        # the call launches on the CURRENT device's current stream; a tensor of another device would be dereferenced there
        raise RuntimeError(f"{name} lives on {t.device} but cuda:{_current_device()} is current: "
                           f"wrap the call in `with torch.cuda.device({t.device.index}):`")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} tensor has to be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"{name} must be {dtype}, got {t.dtype}")
    return t.data_ptr()


def _host_i32(xs: Sequence[int]):
    return (ctypes.c_int32 * len(xs))(*[int(x) for x in xs])


def _host_i64(xs: Sequence[int]):
    return (ctypes.c_int64 * len(xs))(*[int(x) for x in xs])


# ---- MSDA core ------------------------------------------------------------------------------------------
def msda_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, query_order=None, schedule=0):
    """`_C.ms_deform_attn_forward` contract: value (b,Nv,M,D) f32 -> (b,Nq,M*D), fresh tensor."""
    b, nv, m, d = value.shape
    nq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    out = torch.empty(b, nq, m * d, device=value.device, dtype=torch.float32)
    rc = lib().sdetr_msda_forward_ex(
        _req(value, "value", torch.float32), nv * m * d, m * d, _req(spatial_shapes, "spatial_shapes", torch.int64),
        _req(level_start_index, "level_start_index", torch.int64), _req(sampling_loc, "sampling_loc", torch.float32),
        _req(attn_weight, "attn_weight", torch.float32), out.data_ptr(), b, nv, m, d, L, nq, P,
        _req(query_order, "query_order", torch.int32) if query_order is not None else None, schedule, _stream())
    _check(rc, "sdetr_msda_forward_ex")
    return out


def msda_forward_plain(value, spatial_shapes, level_start_index, sampling_loc, attn_weight):
    """The plain entry point (no strides / order), same result as :func:`msda_forward`."""
    b, nv, m, d = value.shape
    nq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    out = torch.empty(b, nq, m * d, device=value.device, dtype=torch.float32)
    rc = lib().sdetr_msda_forward(
        _req(value, "value", torch.float32), _req(spatial_shapes, "spatial_shapes", torch.int64),
        _req(level_start_index, "level_start_index", torch.int64), _req(sampling_loc, "sampling_loc", torch.float32),
        _req(attn_weight, "attn_weight", torch.float32), out.data_ptr(), b, nv, m, d, L, nq, P, _stream())
    _check(rc, "sdetr_msda_forward")
    return out


KERNEL_TIMERS = None  # measurement aid (bench.py): {"msda": [(event_before, event_after), ...]} filled per launch


def _timer_event():
    """CUDA event that can be recorded inside a stream capture AND timed after the graph has run (external event node)."""
    ev = torch.cuda.Event(enable_timing=True, external=torch.cuda.is_current_stream_capturing())
    ev.record()
    return ev


def msda_fused_forward(value_buf, value_batch_stride, value_token_stride, value_offset, spatial_shapes,
                       level_start_index, ref_points, proj, heads, head_dim, levels, points, num_value,
                       query_order=None, schedule=0, want_loc_attn=False):
    """softmax + sampling locations + core in one launch.  ``value_buf`` may be a wide projection buffer;
    ``value_offset`` (floats) selects this layer's column slice.  proj: (b,Nq,>=3*M*L*P) last-dim contiguous."""
    b, nq = proj.shape[0], proj.shape[1]
    if not (proj.is_cuda and proj.stride(2) == 1 and proj.stride(0) == nq * proj.stride(1)):
        raise RuntimeError("proj must be a CUDA tensor with contiguous rows")
    out = torch.empty(b, nq, heads * head_dim, device=proj.device, dtype=torch.float32)
    loc = attn = None
    if want_loc_attn:
        loc = torch.empty(b, nq, heads, levels, points, 2, device=proj.device, dtype=torch.float32)
        attn = torch.empty(b, nq, heads, levels, points, device=proj.device, dtype=torch.float32)
    if not value_buf.is_cuda or value_buf.dtype != torch.float32:
        raise RuntimeError("value must be a CUDA float32 tensor")
    t0 = _timer_event() if KERNEL_TIMERS is not None else None
    if ref_points.shape[-1] not in (2, 4):
        raise ValueError(f"Last dim of reference_points must be 2 or 4, but get {ref_points.shape[-1]} instead.")
    fn = lib().sdetr_msda_fused_forward if ref_points.shape[-1] == 2 else lib().sdetr_msda_fused_forward_boxes
    rc = fn(
        value_buf.data_ptr() + 4 * value_offset, value_batch_stride, value_token_stride,
        _req(spatial_shapes, "spatial_shapes", torch.int64), _req(level_start_index, "level_start_index", torch.int64),
        _req(ref_points, "reference_points", torch.float32), proj.data_ptr(), proj.stride(1), out.data_ptr(),
        loc.data_ptr() if loc is not None else None, attn.data_ptr() if attn is not None else None, b, num_value,
        heads, head_dim, levels, nq, points,
        _req(query_order, "query_order", torch.int32) if query_order is not None else None, schedule, _stream())
    _check(rc, "sdetr_msda_fused_forward")
    if t0 is not None:
        KERNEL_TIMERS.setdefault("msda", []).append((t0, _timer_event()))
    return (out, loc, attn) if want_loc_attn else out


def msda_set_host_shapes(shapes):
    """Level shapes as host integers for the TMA-staged variant's tensor maps (option "msda_tma")."""
    _check(lib().sdetr_msda_set_host_shapes(len(shapes), _host_i32([h for h, _ in shapes]), _host_i32([w for _, w in shapes])),
           "sdetr_msda_set_host_shapes")


def nms_iou_threshold_f32(iou_threshold) -> float:
    """The float32 threshold t32 with `iou > t32` == `iou > iou_threshold` for every float32 IoU: torchvision compares its
    float32 IoU with the double threshold, so a threshold between two floats (1/3 as a Python float) rounds DOWN, never to
    the nearest float (which may be the IoU itself and turn a suppression into a keep)."""
    t = float(iou_threshold)
    t32 = torch.tensor(t, dtype=torch.float32)
    if float(t32) > t:
        t32 = torch.nextafter(t32, torch.tensor(-float("inf")))
    return float(t32)


def nms_topk_index(topk_index, shapes, iou_threshold=0.3):
    """topk_index (b,k) int64, candidates in descending score order -> (kept_index (b,k), kept_count (b,) int32, keep_flag (b,k) u8)."""
    b, k = topk_index.shape
    dev = topk_index.device
    kept = torch.empty(b, k, device=dev, dtype=torch.int64)
    count = torch.empty(b, device=dev, dtype=torch.int32)
    flag = torch.empty(b, k, device=dev, dtype=torch.uint8)
    rc = lib().sdetr_nms_topk_index(_req(topk_index, "topk_index", torch.int64), b, k, sum(h * w for h, w in shapes), len(shapes),
                                    _host_i32([h for h, _ in shapes]), _host_i32([w for _, w in shapes]),
                                    nms_iou_threshold_f32(iou_threshold), kept.data_ptr(), count.data_ptr(), flag.data_ptr(),
                                    _stream())
    _check(rc, "sdetr_nms_topk_index")
    return kept, count, flag


def msda_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output):
    """`_C.ms_deform_attn_backward` contract -> (grad_value, grad_sampling_loc, grad_attn_weight)."""
    b, nv, m, d = value.shape
    nq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    gv = torch.empty_like(value)
    gl = torch.empty_like(sampling_loc)
    ga = torch.empty_like(attn_weight)
    rc = lib().sdetr_msda_backward(
        _req(value, "value", torch.float32), _req(spatial_shapes, "spatial_shapes", torch.int64),
        _req(level_start_index, "level_start_index", torch.int64), _req(sampling_loc, "sampling_loc", torch.float32),
        _req(attn_weight, "attn_weight", torch.float32), _req(grad_output, "grad_output", torch.float32),
        gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), b, nv, m, d, L, nq, P, _stream())
    _check(rc, "sdetr_msda_backward")
    return gv, gl, ga


def msda_backward_deterministic(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output):
    """Same contract as :func:`msda_backward`; grad_value is bit-reproducible (fixed-point accumulation, whatever the order of
    the queries), grad_sampling_loc / grad_attn_weight are bit-identical to msda_backward's.  The int64 accumulator comes from
    the caching allocator (8 bytes per value element)."""
    b, nv, m, d = value.shape
    nq, L, P = sampling_loc.shape[1], sampling_loc.shape[3], sampling_loc.shape[4]
    gv = torch.empty_like(value)
    gl = torch.empty_like(sampling_loc)
    ga = torch.empty_like(attn_weight)
    need = lib().sdetr_msda_backward_deterministic_workspace(b, nv, m, d)
    ws = torch.empty(max(need, 16), device=value.device, dtype=torch.uint8)
    rc = lib().sdetr_msda_backward_deterministic(
        _req(value, "value", torch.float32), _req(spatial_shapes, "spatial_shapes", torch.int64),
        _req(level_start_index, "level_start_index", torch.int64), _req(sampling_loc, "sampling_loc", torch.float32),
        _req(attn_weight, "attn_weight", torch.float32), _req(grad_output, "grad_output", torch.float32),
        gv.data_ptr(), gl.data_ptr(), ga.data_ptr(), b, nv, m, d, L, nq, P, ws.data_ptr(), ws.numel(), _stream())
    _check(rc, "sdetr_msda_backward_deterministic")
    return gv, gl, ga


def upsample_bilinear_ac_backward(grad_fine, Hc: int, Wc: int):
    """Backward of ``F.interpolate(x, size=(H, W), mode="bilinear", align_corners=True)`` for x (..., Hc, Wc):
    grad_fine (..., H, W) -> grad (..., Hc, Wc), deterministic (gather form, no atomics)."""
    H, W = grad_fine.shape[-2:]
    planes = grad_fine.numel() // max(H * W, 1)
    out = torch.empty(*grad_fine.shape[:-2], Hc, Wc, device=grad_fine.device, dtype=torch.float32)
    rc = lib().sdetr_upsample_bilinear_ac_backward(_req(grad_fine, "grad_fine", torch.float32), planes, H, W, Hc, Wc,
                                                   out.data_ptr(), _stream())
    _check(rc, "sdetr_upsample_bilinear_ac_backward")
    return out


# ---- salience filter --------------------------------------------------------------------------------------
def salience_select(raw_score, mask_u8, level_start: Sequence[int], level_size: Sequence[int],
                    level_k: Sequence[int], level_width: Optional[Sequence[int]] = None,
                    level_stride: Optional[Sequence[int]] = None, cell_px: int = 0, workspace=None):
    """-> selected_inds (b,K) i64, selected_score (b,K), foreground_score (b,Nv), tile_order (b,K) i32 | None."""
    b, nv = raw_score.shape
    L = len(level_k)
    K = int(sum(level_k))
    dev = raw_score.device
    inds = torch.empty(b, K, device=dev, dtype=torch.int64)
    score = torch.empty(b, K, device=dev, dtype=torch.float32)
    fg = torch.empty(b, nv, device=dev, dtype=torch.float32)
    want_order = level_width is not None and K > 0
    order = torch.empty(b, K, device=dev, dtype=torch.int32) if want_order else None
    need = lib().sdetr_salience_select_workspace(b, nv, L)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=dev, dtype=torch.uint8)
    rc = lib().sdetr_salience_select(
        _req(raw_score, "raw_score", torch.float32), _req(mask_u8, "mask", torch.uint8), _host_i32(level_start),
        _host_i32(level_size), _host_i32(level_k), _host_i32(level_width) if want_order else None,
        _host_i32(level_stride) if want_order else None, cell_px, b, nv, L, inds.data_ptr(), score.data_ptr(),
        fg.data_ptr(), order.data_ptr() if want_order else None, workspace.data_ptr(), workspace.numel(), _stream())
    _check(rc, "sdetr_salience_select")
    return inds, score, fg, order


def order_prefixes(tile_order, nq_list: Sequence[int]):
    """-> list of (b, nq_j) int32 processing orders, one per encoder layer."""
    b, K = tile_order.shape
    offs, tot = [], 0
    for n in nq_list:
        offs.append(tot)
        tot += b * int(n)
    out = torch.empty(max(tot, 1), device=tile_order.device, dtype=torch.int32)
    rc = lib().sdetr_order_prefixes(_req(tile_order, "tile_order", torch.int32), b, K, len(nq_list),
                                    _host_i32(nq_list), _host_i64(offs), out.data_ptr(), _stream())
    _check(rc, "sdetr_order_prefixes")
    return [out[o:o + b * int(n)].view(b, int(n)) for o, n in zip(offs, nq_list)]


def topk_desc(score, k: int, workspace=None):
    """(segments, n) -> (segments, k) int64 positions of the k largest (ties: smaller position first)."""
    seg, n = score.shape
    out = torch.empty(seg, k, device=score.device, dtype=torch.int64)
    need = lib().sdetr_topk_workspace(seg, n)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, device=score.device, dtype=torch.uint8)
    rc = lib().sdetr_topk_desc(_req(score, "score", torch.float32), seg, n, k, out.data_ptr(), workspace.data_ptr(),
                               workspace.numel(), _stream())
    _check(rc, "sdetr_topk_desc")
    return out


# ---- token movement -----------------------------------------------------------------------------------------
def _inds_view(inds, num_query):
    if not (inds.is_cuda and inds.dtype == torch.int64 and inds.stride(1) == 1 and inds.shape[1] >= num_query):
        raise RuntimeError("inds must be a CUDA int64 tensor with unit column stride")
    return inds.data_ptr(), inds.stride(0)


def token_gather(tokens, pos, fg, valid_ratios, inds, spatial_shapes, level_start_index, num_query, want_sum=False):
    """-> (query, query_pos, fg_q, ref_q[, query + query_pos])"""
    b, nv, c = tokens.shape
    L = spatial_shapes.shape[0]
    dev = tokens.device
    q = torch.empty(b, num_query, c, device=dev, dtype=torch.float32)
    qp = torch.empty(b, num_query, c, device=dev, dtype=torch.float32)
    fq = torch.empty(b, num_query, device=dev, dtype=torch.float32)
    rq = torch.empty(b, num_query, L, 2, device=dev, dtype=torch.float32)
    qs = torch.empty(b, num_query, c, device=dev, dtype=torch.float32) if want_sum else None
    ip, istride = _inds_view(inds, num_query)
    rc = lib().sdetr_token_gather(
        _req(tokens, "tokens", torch.float32), _req(pos, "pos", torch.float32), _req(fg, "fg", torch.float32),
        _req(valid_ratios, "valid_ratios", torch.float32), ip, istride, _req(spatial_shapes, "spatial_shapes", torch.int64),
        _req(level_start_index, "level_start_index", torch.int64), b, nv, c, L, num_query, q.data_ptr(), qp.data_ptr(),
        fq.data_ptr(), rq.data_ptr(), qs.data_ptr() if want_sum else None, _stream())
    _check(rc, "sdetr_token_gather")
    return (q, qp, fq, rq, qs) if want_sum else (q, qp, fq, rq)


def token_scatter_(tokens, query, inds, focus_token_nums):
    b, nv, c = tokens.shape
    nq = query.shape[1]
    ip, istride = _inds_view(inds, nq)
    rc = lib().sdetr_token_scatter(_req(tokens, "tokens", torch.float32), _req(query, "query", torch.float32), ip,
                                   istride, _req(focus_token_nums, "focus_token_nums", torch.int32), b, nv, c, nq,
                                   _stream())
    _check(rc, "sdetr_token_scatter")
    return tokens


def background_embed_(tokens, mask_u8, last_inds, row_embed, col_embed, spatial_shapes, level_start_index, flags=None,
                      shapes_host: Optional[Sequence[Sequence[int]]] = None):
    """``shapes_host``: the [(H, W), ...] of the levels as host ints; a map larger than the embedding tables then raises
    like the reference's ``nn.Embedding`` lookup.  Without it the shapes are fetched from the device (one sync)."""
    b, nv, c = tokens.shape
    num_last = last_inds.shape[1]
    ip, istride = _inds_view(last_inds, num_last)
    if flags is None:
        flags = torch.empty(b, nv, device=tokens.device, dtype=torch.uint8)
    L = spatial_shapes.shape[0]
    if shapes_host is None:
        shapes_host = spatial_shapes.tolist()
    host = (ctypes.c_int64 * (2 * L))(*[int(v) for hw in shapes_host for v in hw])
    rc = lib().sdetr_background_embed(
        _req(tokens, "tokens", torch.float32), _req(mask_u8, "mask", torch.uint8), ip, istride, num_last,
        _req(row_embed, "row_embed", torch.float32), _req(col_embed, "col_embed", torch.float32),
        min(row_embed.shape[0], col_embed.shape[0]),
        _req(spatial_shapes, "spatial_shapes", torch.int64), ctypes.cast(host, ctypes.c_void_p),
        _req(level_start_index, "level_start_index", torch.int64),
        b, nv, c, L, _req(flags, "flags", torch.uint8), _stream())
    _check(rc, "sdetr_background_embed")
    return tokens


def score_modulate(mem_all, level_start: int, H: int, W: int, coarse_score, Hc: int, Wc: int, alpha, alpha_index: int):
    """mem_all (b,Nv,C) contiguous; the level slice starts at token ``level_start``.  coarse_score (b,Hc*Wc) rows
    (any batch stride).  -> (b,H*W,C)."""
    b, nv, c = mem_all.shape
    out = torch.empty(b, H * W, c, device=mem_all.device, dtype=torch.float32)
    if not (coarse_score.is_cuda and coarse_score.stride(1) == 1 and coarse_score.dtype == torch.float32):
        raise RuntimeError("coarse_score rows must be contiguous CUDA float32")
    if not 0 <= alpha_index < alpha.numel():  # the reference raises IndexError on alpha[lvl] (salience_transformer.py:143)
        raise IndexError(f"alpha has {alpha.numel()} entries, level {alpha_index} asked for")
    rc = lib().sdetr_score_modulate(
        _req(mem_all, "mem", torch.float32) + 4 * level_start * c, nv * c, coarse_score.data_ptr(),
        coarse_score.stride(0), _req(alpha, "alpha", torch.float32), alpha_index, b, H, W, Hc, Wc, c, out.data_ptr(),
        _stream())
    _check(rc, "sdetr_score_modulate")
    return out


def mask_predictor_level(mem_all, level_start: int, H: int, W: int, coarse_score, Hc: int, Wc: int, alpha, alpha_index: int,
                         ln_gamma, ln_beta, eps: float, w1_t, b1, w2a_t, b2a, w2b_t, b2b, w2c, b2c, raw, out_start: int):
    """Score modulation + MaskPredictor of one level in two launches.  mem_all (b,Nv,256) contiguous, the level's tokens start at
    ``level_start``; coarse_score: (b,Hc*Wc) rows of the next coarser level's raw scores (any batch stride) or None; weights
    transposed to (in, out); writes raw[:, out_start:out_start + H*W] (raw (b,Nv) contiguous)."""
    b, nv, c = mem_all.shape
    if coarse_score is not None:
        if not (coarse_score.is_cuda and coarse_score.stride(1) == 1 and coarse_score.dtype == torch.float32):
            raise RuntimeError("coarse_score rows must be contiguous CUDA float32")
        if not 0 <= alpha_index < alpha.numel():
            raise IndexError(f"alpha has {alpha.numel()} entries, level {alpha_index} asked for")
    if not (raw.is_cuda and raw.dtype == torch.float32 and raw.is_contiguous() and tuple(raw.shape) == (b, nv)):
        raise RuntimeError("raw must be a contiguous CUDA float32 (b, Nv) tensor")
    ws = torch.empty(int(lib().sdetr_mask_predictor_level_workspace_floats(b, H, W)), device=mem_all.device, dtype=torch.float32)
    rc = lib().sdetr_mask_predictor_level(
        _req(mem_all, "mem", torch.float32) + 4 * level_start * c, nv * c, b, H, W, c,
        coarse_score.data_ptr() if coarse_score is not None else None, coarse_score.stride(0) if coarse_score is not None else 0,
        Hc, Wc, _req(alpha, "alpha", torch.float32) if coarse_score is not None else None, alpha_index,
        _req(ln_gamma, "ln_gamma", torch.float32), _req(ln_beta, "ln_beta", torch.float32), float(eps),
        _req(w1_t, "w1_t", torch.float32), _req(b1, "b1", torch.float32), _req(w2a_t, "w2a_t", torch.float32),
        _req(b2a, "b2a", torch.float32), _req(w2b_t, "w2b_t", torch.float32), _req(b2b, "b2b", torch.float32),
        _req(w2c, "w2c", torch.float32), _req(b2c, "b2c", torch.float32), ws.data_ptr(), ws.numel(),
        raw.data_ptr() + 4 * out_start, nv, _stream())
    _check(rc, "sdetr_mask_predictor_level")
    return raw


def zero_masked_rows_(buf, row_stride: int, row_floats: int, mask_u8, num_rows: int, offset_floats: int = 0):
    rc = lib().sdetr_zero_masked_rows(buf.data_ptr() + 4 * offset_floats, row_stride, row_floats,
                                      _req(mask_u8, "mask", torch.uint8), num_rows, _stream())
    _check(rc, "sdetr_zero_masked_rows")
    return buf


def class_max_times_fg(logits, fg):
    """logits (..., num_classes) with unit last stride and a uniform row pitch (a padded GEMM output is fine)."""
    rows = fg.numel()
    out = torch.empty_like(fg)
    if not (logits.is_cuda and logits.dtype == torch.float32 and logits.stride(-1) == 1):
        raise RuntimeError("logits must be CUDA float32 with unit last stride")
    pitch = logits.stride(-2)
    if logits.dim() == 3 and logits.stride(0) != logits.shape[1] * pitch:
        logits, pitch = logits.contiguous(), logits.shape[-1]
    rc = lib().sdetr_class_max_times_fg(logits.data_ptr(), pitch, _req(fg, "fg", torch.float32), rows,
                                        logits.shape[-1], out.data_ptr(), _stream())
    _check(rc, "sdetr_class_max_times_fg")
    return out


def add_layernorm(x, r, gamma, beta, eps: float = 1e-5, out=None):
    """LayerNorm(x + r); r may be None; out may alias x."""
    c = x.shape[-1]
    rows = x.numel() // c
    if out is None:
        out = torch.empty_like(x)
    rc = lib().sdetr_add_layernorm(_req(x, "x", torch.float32), _req(r, "r", torch.float32) if r is not None else None,
                                   _req(gamma, "gamma", torch.float32), _req(beta, "beta", torch.float32), eps, rows, c,
                                   out.data_ptr(), _stream())
    _check(rc, "sdetr_add_layernorm")
    return out


def split_tf32(x, layout_b: bool = False, relu=0, chunk: int = 0):
    """(..., K) fp32 with contiguous rows -> (rows, 3K) 3xTF32 operand: per K-chunk [hi|hi|lo] (weights: [hi|lo|hi])."""
    K = x.shape[-1]
    chunk = chunk or K
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("split_tf32 needs a CUDA float32 tensor with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)  # view when rows are uniformly strided
    rows = x2.shape[0]
    out = torch.empty(rows, 3 * K, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_split_tf32(x2.data_ptr(), x2.stride(0) if rows > 1 else K, rows, K, chunk, int(layout_b), int(relu),
                                out.data_ptr(), _stream())
    _check(rc, "sdetr_split_tf32")
    return out


def rows_scatter_(dst, index, src):
    """dst (b,n,C) <- src (b,k,C) at index (b,k) int64, in place."""
    b, n, c = dst.shape
    k = index.shape[1]
    rc = lib().sdetr_rows_scatter(_req(dst, "dst", torch.float32), _req(index, "index", torch.int64), b, n, k, c,
                                  _req(src, "src", torch.float32), _stream())
    _check(rc, "sdetr_rows_scatter")
    return dst


def split_tf32_pair(w):
    """(N,K) fp32 -> (W_hi, W_lo), both TF32-representable fp32 tensors of the same shape."""
    w = w.contiguous()
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    _check(lib().sdetr_split_tf32_pair(_req(w, "w", torch.float32), w.numel(), hi.data_ptr(), lo.data_ptr(), _stream()),
           "sdetr_split_tf32_pair")
    return hi, lo


def gemm_3xtf32(x, w_hi, w_lo, bias=None, relu_input=0):
    """y = act(x) @ W.T + bias on the wgmma tensor cores; x (..., K) with unit last stride and uniform row pitch."""
    K = x.shape[-1]
    N = w_hi.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_3xtf32 needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    y = torch.empty(M, N, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_3xtf32(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w_hi, "w_hi", torch.float32),
                                 _req(w_lo, "w_lo", torch.float32),
                                 _req(bias, "bias", torch.float32) if bias is not None else None, y.data_ptr(), N, M, N, K,
                                 int(relu_input), _stream())
    _check(rc, "sdetr_gemm_3xtf32")
    return y.view(*x.shape[:-1], N)


def flatten_tokens(feats, pos, level_embeds, keep):
    """Per-level (b,C,H,W) feats / pos -> (feat_tok, lpos_tok, x_tok), each (b,Nv,C); keep (b,Nv) float."""
    L = len(feats)
    b, c = feats[0].shape[:2]
    sizes = [f.shape[2] * f.shape[3] for f in feats]
    nv = sum(sizes)
    dev = feats[0].device
    fp = (ctypes.c_void_p * L)(*[_req(f, "feat", torch.float32) for f in feats])
    pp = (ctypes.c_void_p * L)(*[_req(p, "pos", torch.float32) for p in pos])
    out = [torch.empty(b, nv, c, device=dev, dtype=torch.float32) for _ in range(3)]
    rc = lib().sdetr_flatten_tokens(fp, pp, _req(level_embeds, "level_embeds", torch.float32), _req(keep, "keep", torch.float32),
                                    _host_i32(sizes), b, c, L, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), _stream())
    _check(rc, "sdetr_flatten_tokens")
    return out


def flatten_tokens_pos(feats, pos_tokens, level_embeds, keep):
    """Per-level (b,C,H,W) feats + token-layout position embedding (b,Nv,C) -> (feat_tok, lpos_tok, x_tok)."""
    L = len(feats)
    b, c = feats[0].shape[:2]
    sizes = [f.shape[2] * f.shape[3] for f in feats]
    nv = sum(sizes)
    fp = (ctypes.c_void_p * L)(*[_req(f, "feat", torch.float32) for f in feats])
    out = [torch.empty(b, nv, c, device=feats[0].device, dtype=torch.float32) for _ in range(3)]
    if tuple(pos_tokens.shape) != (b, nv, c):
        raise RuntimeError(f"pos_tokens must be {(b, nv, c)}, got {tuple(pos_tokens.shape)}")
    rc = lib().sdetr_flatten_tokens_pos(fp, _req(pos_tokens, "pos_tokens", torch.float32),
                                        _req(level_embeds, "level_embeds", torch.float32), _req(keep, "keep", torch.float32),
                                        _host_i32(sizes), b, c, L, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), _stream())
    _check(rc, "sdetr_flatten_tokens_pos")
    return out


def salience_targets(boxes_xyxy, num_boxes, shapes, strides, limit_range):
    """boxes (b,max_boxes,4) xyxy pixels (padded), num_boxes (b,) int32 -> (b,Nv) salience targets (noise-free)."""
    b, mb = boxes_xyxy.shape[:2]
    nv = sum(h * w for h, w in shapes)
    out = torch.empty(b, nv, device=num_boxes.device, dtype=torch.float32)
    f = lambda xs: (ctypes.c_float * len(xs))(*[float(x) for x in xs])  # noqa: E731
    rc = lib().sdetr_salience_targets(_req(boxes_xyxy, "boxes", torch.float32) if mb else None, _req(num_boxes, "num_boxes", torch.int32),
                                      mb, b, nv, len(shapes), _host_i32([h for h, _ in shapes]), _host_i32([w for _, w in shapes]),
                                      f([s[0] for s in strides]), f([s[1] for s in strides]), f([r[0] for r in limit_range]),
                                      f([r[1] for r in limit_range]), out.data_ptr(), _stream())
    _check(rc, "sdetr_salience_targets")
    return out


def tokens_to_maps(tokens, shapes):
    """(b,Nv,C) tokens -> list of per-level (b,C,H,W) maps (one launch; salience_transformer.py:186-190)."""
    b, nv, c = tokens.shape
    maps = [torch.empty(b, c, h, w, device=tokens.device, dtype=torch.float32) for h, w in shapes]
    ptrs = (ctypes.c_void_p * len(shapes))(*[m.data_ptr() for m in maps])
    rc = lib().sdetr_token_map_transpose(_req(tokens, "tokens", torch.float32), ptrs, _host_i32([h * w for h, w in shapes]), b, c,
                                         len(shapes), 1, _stream())
    _check(rc, "sdetr_token_map_transpose")
    return maps


def maps_to_tokens(maps):
    """list of per-level (b,C,H,W) maps -> (b,Nv,C) tokens (one launch; salience_transformer.py:192)."""
    b, c = maps[0].shape[:2]
    sizes = [m.shape[2] * m.shape[3] for m in maps]
    tokens = torch.empty(b, sum(sizes), c, device=maps[0].device, dtype=torch.float32)
    ptrs = (ctypes.c_void_p * len(maps))(*[_req(m, "map", torch.float32) for m in maps])
    rc = lib().sdetr_token_map_transpose(tokens.data_ptr(), ptrs, _host_i32(sizes), b, c, len(maps), 0, _stream())
    _check(rc, "sdetr_token_map_transpose")
    return tokens


def mask_plan(mask_u8, shapes, level_filter_ratio, pos_offset=-0.5, pos_eps=1e-6, pos_scale=2 * 3.141592653589793):
    """mask_u8 (b,Nv) -> dict(valid (b,L) i32, focus (b,L) i32, valid_ratios (b,L,2), keep (b,Nv), ynorm, xnorm (b,Nv))."""
    b, nv = mask_u8.shape
    L = len(shapes)
    dev = mask_u8.device
    f32 = dict(device=dev, dtype=torch.float32)
    out = dict(valid=torch.empty(b, L, device=dev, dtype=torch.int32), focus=torch.empty(b, L, device=dev, dtype=torch.int32),
               valid_ratios=torch.empty(b, L, 2, **f32), keep=torch.empty(b, nv, **f32), ynorm=torch.empty(b, nv, **f32),
               xnorm=torch.empty(b, nv, **f32))
    ratios = (ctypes.c_float * L)(*[float(r) for r in level_filter_ratio])
    rc = lib().sdetr_mask_plan(_req(mask_u8, "mask", torch.uint8), b, nv, L, _host_i32([h for h, _ in shapes]),
                               _host_i32([w for _, w in shapes]), ratios, float(pos_offset), float(pos_eps), float(pos_scale),
                               out["ynorm"].data_ptr(), out["xnorm"].data_ptr(), out["valid"].data_ptr(), out["focus"].data_ptr(),
                               out["valid_ratios"].data_ptr(), out["keep"].data_ptr(), _stream())
    _check(rc, "sdetr_mask_plan")
    return out


def sine_pos_tokens(ynorm, xnorm, dim_ty, dim_tx):
    """(b,Nv) normalised coordinates -> (b,Nv,2F) sine position embedding in token layout."""
    b, nv = ynorm.shape
    f = dim_ty.numel()
    pos = torch.empty(b, nv, 2 * f, device=ynorm.device, dtype=torch.float32)
    rc = lib().sdetr_sine_pos_tokens(_req(ynorm, "ynorm", torch.float32), _req(xnorm, "xnorm", torch.float32),
                                     _req(dim_ty, "dim_ty", torch.float32), _req(dim_tx, "dim_tx", torch.float32), b * nv, f,
                                     pos.data_ptr(), _stream())
    _check(rc, "sdetr_sine_pos_tokens")
    return pos


def gemm_3xtf32_raw(x, w, bias=None, act=0):
    """y = act(x) @ w.T + bias, both operands split inside the kernel (w: raw fp32 (N,K) contiguous)."""
    K = x.shape[-1]
    N = w.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_3xtf32_raw needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    ldc = (N + 3) // 4 * 4  # 16-byte row pitch lets the epilogue leave through TMA bulk stores (e.g. N = 91 -> 92)
    y = torch.empty(M, ldc, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_3xtf32_raw(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w, "w", torch.float32),
                                     _req(bias, "bias", torch.float32) if bias is not None else None, y.data_ptr(), ldc, M, N, K,
                                     int(act), _stream())
    _check(rc, "sdetr_gemm_3xtf32_raw")
    y = y if ldc == N else y[:, :N]
    return y.reshape(*x.shape[:-1], N) if ldc == N else y.unflatten(0, x.shape[:-1])


def gemm_3xtf32_pre(x, w_hi, w_lo, bias=None, act=0):
    """y = act(x) @ (w_hi + w_lo).T + bias on the persistent kernel with a pre-split weight (sdetr_split_tf32_pair)."""
    K = x.shape[-1]
    N = w_hi.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_3xtf32_pre needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    ldc = (N + 3) // 4 * 4
    y = torch.empty(M, ldc, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_3xtf32_pre(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w_hi, "w_hi", torch.float32),
                                     _req(w_lo, "w_lo", torch.float32),
                                     _req(bias, "bias", torch.float32) if bias is not None else None, y.data_ptr(), ldc, M, N, K,
                                     int(act), _stream())
    _check(rc, "sdetr_gemm_3xtf32_pre")
    y = y if ldc == N else y[:, :N]
    return y.reshape(*x.shape[:-1], N) if ldc == N else y.unflatten(0, x.shape[:-1])


def split_f16_pair(w):
    """(N,K) fp32 -> (W_hi, W_lo, scale): fp16 pair of scale * W with scale = 2^s such that max|scale * W| is in
    [2^13, 2^14) (one host read of max|W|; done once per parameter version by gemm.split_weight_f16)."""
    import math
    w = w.contiguous()
    amax = float(w.abs().max())
    if not math.isfinite(amax):
        raise RuntimeError("split_f16_pair: weight has non-finite entries")
    scale = 2.0 ** (13 - math.frexp(amax)[1] + 1) if amax > 0 else 1.0  # frexp: amax = m * 2^e, 0.5 <= m < 1
    hi = torch.empty(w.shape, device=w.device, dtype=torch.float16)
    lo = torch.empty_like(hi)
    _check(lib().sdetr_split_f16_pair(_req(w, "w", torch.float32), w.numel(), scale, hi.data_ptr(), lo.data_ptr(), _stream()),
           "sdetr_split_f16_pair")
    return hi, lo, scale


def gemm_f16x3_pre(x, w_hi, w_lo, w_scale, bias=None, act=0, out=None):
    """y = act(x) @ W.T + bias on the persistent wgmma .f16 kernel (3xFP16, fp32-class accuracy).
    ``out``: optional (M, N) fp32 destination with unit column stride (e.g. a row slice of a larger buffer)."""
    K = x.shape[-1]
    N = w_hi.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_f16x3_pre needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    if out is not None:
        if not (out.is_cuda and out.dtype == torch.float32 and out.dim() == 2 and tuple(out.shape) == (M, N) and out.stride(1) == 1):
            raise RuntimeError(f"gemm_f16x3_pre: out must be a CUDA float32 ({M}, {N}) tensor with unit column stride")
        rc = lib().sdetr_gemm_f16x3_pre(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w_hi, "w_hi", torch.float16),
                                        _req(w_lo, "w_lo", torch.float16), float(w_scale),
                                        _req(bias, "bias", torch.float32) if bias is not None else None, out.data_ptr(),
                                        out.stride(0) if M > 1 else N, M, N, K, int(act), _stream())
        _check(rc, "sdetr_gemm_f16x3_pre")
        return out
    ldc = (N + 3) // 4 * 4
    y = torch.empty(M, ldc, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_f16x3_pre(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w_hi, "w_hi", torch.float16),
                                    _req(w_lo, "w_lo", torch.float16), float(w_scale),
                                    _req(bias, "bias", torch.float32) if bias is not None else None, y.data_ptr(), ldc, M, N, K,
                                    int(act), _stream())
    _check(rc, "sdetr_gemm_f16x3_pre")
    y = y if ldc == N else y[:, :N]
    return y.reshape(*x.shape[:-1], N) if ldc == N else y.unflatten(0, x.shape[:-1])


def gemm_f16x3_rowmax(x, w_hi, w_lo, w_scale, bias, row_scale):
    """max over the N <= 128 columns of (x @ W.T + bias), times row_scale, per row of x (..., K): bit for bit
    ``class_max_times_fg(gemm_f16x3_pre(x, w_hi, w_lo, w_scale, bias), row_scale)`` in one launch.  -> x.shape[:-1]"""
    K = x.shape[-1]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_f16x3_rowmax needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    rs = _req(row_scale, "row_scale", torch.float32)
    if row_scale.numel() != M:
        raise RuntimeError(f"gemm_f16x3_rowmax: row_scale must hold one value per row ({M})")
    out = torch.empty(x.shape[:-1], device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_f16x3_rowmax(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(w_hi, "w_hi", torch.float16),
                                       _req(w_lo, "w_lo", torch.float16), float(w_scale),
                                       _req(bias, "bias", torch.float32) if bias is not None else None, rs, out.data_ptr(),
                                       M, w_hi.shape[0], K, _stream())
    _check(rc, "sdetr_gemm_f16x3_rowmax")
    return out


def gemm_f16x3_add_layernorm_(q, x, w_hi, w_lo, w_scale, bias, gamma, beta, eps: float = 1e-5):
    """q = LayerNorm(q + x @ W.T + bias) * gamma + beta in place, W (256, 256) as a ``split_f16_pair`` triple: bit for bit
    ``add_layernorm(q, gemm_f16x3_pre(x, ...), gamma, beta, eps, out=q)`` in one launch.  q (..., 256) contiguous, x of the
    same rows with unit last stride."""
    if not (q.is_cuda and q.dtype == torch.float32 and q.shape[-1] == 256 and q.is_contiguous()):
        raise RuntimeError("gemm_f16x3_add_layernorm_ needs a contiguous CUDA float32 (..., 256) q")
    if not (x.is_cuda and x.dtype == torch.float32 and x.shape[-1] == 256 and x.stride(-1) == 1):
        raise RuntimeError("gemm_f16x3_add_layernorm_ needs a CUDA float32 (..., 256) x with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, 256)
    M = x2.shape[0]
    if q.numel() != M * 256 or tuple(w_hi.shape) != (256, 256):
        raise RuntimeError("gemm_f16x3_add_layernorm_: q and x must have the same rows, W must be (256, 256)")
    rc = lib().sdetr_gemm_f16x3_add_layernorm(
        x2.data_ptr(), x2.stride(0) if M > 1 else 256, _req(w_hi, "w_hi", torch.float16), _req(w_lo, "w_lo", torch.float16),
        float(w_scale), _req(bias, "bias", torch.float32) if bias is not None else None, _req(gamma, "gamma", torch.float32),
        _req(beta, "beta", torch.float32), float(eps), q.data_ptr(), M, _stream())
    _check(rc, "sdetr_gemm_f16x3_add_layernorm")
    return q


def ffn_fused_layernorm(x, w1, b1, w2, b2, gamma=None, beta=None, eps: float = 1e-5, out=None):
    """y = LayerNorm(x + linear2(ReLU(linear1(x)))) by the 3xFP16 wgmma kernel (gamma None: the bare FFN, no residual / norm).
    ``w1`` / ``w2``: (W_hi, W_lo, scale) triples of ``split_f16_pair``; x (..., 256) fp32 with unit last stride."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.shape[-1] == 256 and x.stride(-1) == 1):
        raise RuntimeError("ffn_fused_layernorm needs a CUDA float32 (..., 256) input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, 256)
    M = x2.shape[0]
    hidden = w1[0].shape[0]
    if tuple(w1[0].shape) != (hidden, 256) or tuple(w2[0].shape) != (256, hidden):
        raise RuntimeError("ffn_fused_layernorm: W1 must be (hidden, 256) and W2 (256, hidden)")
    y = out if out is not None else torch.empty(M, 256, device=x.device, dtype=torch.float32)
    if not (y.is_cuda and y.dtype == torch.float32 and y.is_contiguous() and y.numel() == M * 256):
        raise RuntimeError("ffn_fused_layernorm: out must be a contiguous CUDA float32 tensor of the input's size")
    ws = torch.empty(max(int(lib().sdetr_ffn_fused_workspace_floats(M, hidden)), 4), device=x.device, dtype=torch.float32)
    rc = lib().sdetr_ffn_fused_layernorm(
        x2.data_ptr(), x2.stride(0) if M > 1 else 256, _req(w1[0], "w1_hi", torch.float16), _req(w1[1], "w1_lo", torch.float16),
        float(w1[2]), _req(b1, "b1", torch.float32), _req(w2[0], "w2_hi", torch.float16), _req(w2[1], "w2_lo", torch.float16),
        float(w2[2]), _req(b2, "b2", torch.float32) if b2 is not None else None,
        _req(gamma, "gamma", torch.float32) if gamma is not None else None,
        _req(beta, "beta", torch.float32) if beta is not None else None, float(eps), M, hidden, ws.data_ptr(), ws.numel(),
        y.data_ptr(), _stream())
    _check(rc, "sdetr_ffn_fused_layernorm")
    return y if out is not None else y.reshape(x.shape)


_pow2_state = {}


def pow2_scale(x, target_log2: int = 12):
    """Device scalar 2^s with max|x| * 2^s in [2^(target_log2 - 1), 2^target_log2); no host synchronisation."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
        raise RuntimeError("pow2_scale needs a contiguous CUDA float32 tensor")
    key = (x.device.index, _stream())
    st = _pow2_state.get(key)
    if st is None:
        st = _pow2_state[key] = torch.zeros(2, device=x.device, dtype=torch.int32)  # per (device, stream): calls are stream-ordered
    out = torch.empty(1, device=x.device, dtype=torch.float32)
    _check(lib().sdetr_pow2_scale(x.data_ptr(), x.numel(), int(target_log2), st.data_ptr(), out.data_ptr(), _stream()), "sdetr_pow2_scale")
    return out


def split_f16_pair_dev(w, scale=None):
    """(W_hi, W_lo, scale) with the power-of-two scale computed and kept ON THE DEVICE (training: the weights change every step)."""
    w = w if w.is_contiguous() else w.contiguous()
    scale = pow2_scale(w, 14) if scale is None else scale
    hi = torch.empty(w.shape, device=w.device, dtype=torch.float16)
    lo = torch.empty_like(hi)
    _check(lib().sdetr_split_f16_pair_dev(_req(w, "w", torch.float32), w.numel(), scale.data_ptr(), hi.data_ptr(), lo.data_ptr(), _stream()),
           "sdetr_split_f16_pair_dev")
    return hi, lo, scale


def gemm_f16x3_scaled(x, a_scale, w_hi, w_lo, w_scale, bias=None):
    """y = x @ W.T + bias; ``a_scale`` / ``w_scale``: device scalars (pow2_scale / split_f16_pair_dev) -- no host synchronisation."""
    K = x.shape[-1]
    N = w_hi.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_f16x3_scaled needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    ldc = (N + 3) // 4 * 4
    # the result must not be a view (autograd Functions hand it out, and in-place ops on it are legal): final shape when N % 4 == 0
    y = torch.empty(*x.shape[:-1], N, device=x.device, dtype=torch.float32) if ldc == N else torch.empty(M, ldc, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_gemm_f16x3_scaled(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(a_scale, "a_scale", torch.float32),
                                       _req(w_hi, "w_hi", torch.float16), _req(w_lo, "w_lo", torch.float16),
                                       _req(w_scale, "w_scale", torch.float32),
                                       _req(bias, "bias", torch.float32) if bias is not None else None, y.data_ptr(), ldc, M, N, K,
                                       _stream())
    _check(rc, "sdetr_gemm_f16x3_scaled")
    return y if ldc == N else y[:, :N].contiguous().reshape(*x.shape[:-1], N)


def rows_gather_add(src, pos, index):
    """t = src[b, index], x = t + pos[b, index]  (the pre-attention's two gathers and the `with_pos_embed` add)."""
    b, n, c = src.shape
    k = index.shape[1]
    t = torch.empty(b, k, c, device=src.device, dtype=torch.float32)
    x = torch.empty_like(t)
    rc = lib().sdetr_rows_gather_add(_req(src, "src", torch.float32), _req(pos, "pos", torch.float32),
                                     _req(index, "index", torch.int64), b, n, k, c, t.data_ptr(), x.data_ptr(), _stream())
    _check(rc, "sdetr_rows_gather_add")
    return t, x


def attention_qkv(qkv, heads: int):
    """qkv (b,n,3C) packed [q | k | v] projections -> (b,n,C) = softmax(QK^T/sqrt(d)) V per head (d = C/heads = 32)."""
    b, n, c3 = qkv.shape
    c = c3 // 3
    out = torch.empty(b, n, c, device=qkv.device, dtype=torch.float32)
    rc = lib().sdetr_attention_qkv(_req(qkv, "qkv", torch.float32), out.data_ptr(), b, n, heads, c // heads, _stream())
    _check(rc, "sdetr_attention_qkv")
    return out


def mha_in_proj(tokens, pos, index, w_in_t, b_in):
    """tokens/pos (b,nq,C), index (b,k) int64, w_in_t (C,3C) = in_proj_weight.T -> (t (b,k,C), qkv (b,k,3C))."""
    b, nq, c = tokens.shape
    k = index.shape[1]
    t = torch.empty(b, k, c, device=tokens.device, dtype=torch.float32)
    qkv = torch.empty(b, k, 3 * c, device=tokens.device, dtype=torch.float32)
    if tuple(w_in_t.shape) != (c, 3 * c) or b_in.numel() != 3 * c:
        raise RuntimeError("w_in_t must be (C, 3C) and b_in (3C)")
    rc = lib().sdetr_mha_in_proj(_req(tokens, "tokens", torch.float32), _req(pos, "pos", torch.float32),
                                 _req(index, "index", torch.int64), b, nq, k, c, _req(w_in_t, "w_in_t", torch.float32),
                                 _req(b_in, "b_in", torch.float32), t.data_ptr(), qkv.data_ptr(), _stream())
    _check(rc, "sdetr_mha_in_proj")
    return t, qkv


def mha_out_proj_ln_scatter_(dst, attn, t, w_out_t, b_out, gamma, beta, eps: float, index, pos=None, dst_sum=None):
    """dst (b,nq,C) <- LayerNorm(t + attn @ w_out_t + b_out) at index (b,k), in place; with pos / dst_sum (b,nq,C) the
    same rows of dst_sum receive the new row + pos."""
    b, nq, c = dst.shape
    k = index.shape[1]
    if tuple(w_out_t.shape) != (c, c):
        raise RuntimeError("w_out_t must be (C, C)")
    rc = lib().sdetr_mha_out_proj_ln_scatter(
        _req(attn, "attn", torch.float32), _req(t, "t", torch.float32), _req(w_out_t, "w_out_t", torch.float32),
        _req(b_out, "b_out", torch.float32), _req(gamma, "gamma", torch.float32), _req(beta, "beta", torch.float32),
        float(eps), _req(index, "index", torch.int64), _req(dst, "dst", torch.float32),
        _req(pos, "pos", torch.float32) if pos is not None else None,
        _req(dst_sum, "dst_sum", torch.float32) if dst_sum is not None else None, b, nq, k, c, _stream())
    _check(rc, "sdetr_mha_out_proj_ln_scatter")
    return dst


def gelu_colmean_(z, half: int):
    """z (b,n,C) in place: GELU everywhere, then columns [half, C) replaced by their per-image token mean."""
    b, n, c = z.shape
    need = lib().sdetr_gelu_colmean_workspace(b, n, c, half)
    ws = torch.empty(need, device=z.device, dtype=torch.uint8)
    rc = lib().sdetr_gelu_colmean(_req(z, "z", torch.float32), b, n, c, half, ws.data_ptr(), ws.numel(), _stream())
    _check(rc, "sdetr_gelu_colmean")
    return z


# ---- RepVGG-PluX neck in token layout (neck.RepVGGPluXNetwork.forward_tokens) --------------------------------------------
def _token_rows(t, name):
    """(b, HW, C) fp32 CUDA view with unit channel stride -> (pointer, image pitch, row stride) in floats"""
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 3 and t.stride(2) == 1):
        raise RuntimeError(f"{name} must be a CUDA float32 (b, HW, C) tensor with unit channel stride")
    if t.device.index != _current_device():
        raise RuntimeError(f"{name} lives on {t.device} but cuda:{_current_device()} is current")
    return t.data_ptr(), t.stride(0), t.stride(1)


ACT_RELU, ACT_SILU = 1, 3


def conv2d_f16x3(x, hw, a_scale, w_hi, w_lo, w_scale, bias, groups: int, ksize: int, stride: int, act: int = 0, out=None, z=None):
    """y = act(conv2d(x, W) + bias (+ z)) on token rows.  x: (b, H*W, Cin) view (e.g. a level slice of the encoder memory), hw = (H, W);
    W given as the (Cout, k, k, Cin / groups) pair of split_f16_pair_dev and its device scale; a_scale: pow2_scale of x (target 12).
    act: 0, ACT_RELU or ACT_SILU.  z: optional (b, Ho*Wo, Cout) residual view, may be ``out`` itself.
    out: optional (b, Ho*Wo, Cout) view to write; returns it (or a new contiguous tensor)."""
    H, W = hw
    b, hw_in, cin = x.shape
    if hw_in != H * W:
        raise RuntimeError(f"conv2d_f16x3: x has {hw_in} rows per image, the map is {H}x{W}")
    cout = w_hi.shape[0]
    pad = ksize // 2
    ho, wo = (H + 2 * pad - ksize) // stride + 1, (W + 2 * pad - ksize) // stride + 1
    y = out if out is not None else torch.empty(b, ho * wo, cout, device=x.device, dtype=torch.float32)
    if tuple(y.shape) != (b, ho * wo, cout):
        raise RuntimeError(f"conv2d_f16x3: out must be ({b}, {ho * wo}, {cout})")
    if z is not None and tuple(z.shape) != (b, ho * wo, cout):
        raise RuntimeError(f"conv2d_f16x3: z must be ({b}, {ho * wo}, {cout})")
    xp, xpitch, ldx = _token_rows(x, "x")
    yp, ypitch, ldy = _token_rows(y, "out")
    zp = _token_rows(z, "z") if z is not None else (None, 0, 0)
    rc = lib().sdetr_conv2d_f16x3(xp, xpitch, ldx, b, H, W, cin, _req(a_scale, "a_scale", torch.float32),
                                  _req(w_hi, "w_hi", torch.float16), _req(w_lo, "w_lo", torch.float16),
                                  _req(w_scale, "w_scale", torch.float32),
                                  _req(bias, "bias", torch.float32) if bias is not None else None, *zp, cout, int(groups),
                                  int(ksize), int(stride), int(act), yp, ypitch, ldy, _stream())
    _check(rc, "sdetr_conv2d_f16x3")
    return y


def context_gate(y, x, w_mask, b_mask, w1, w2, z=None, out=None):
    """out = sigmoid(W2 ReLU(W1 ctx)) * y + x (+ z), ctx = softmax over each image's pixels of (y . w_mask + b_mask) . y.
    y, x, z, out: (b, HW, C) views; w_mask (C), b_mask (1) device tensors, w1 (C / r, C), w2 (C, C / r)."""
    b, hw, c = y.shape
    r = w1.shape[0]
    out = out if out is not None else torch.empty(b, hw, c, device=y.device, dtype=torch.float32)
    ops = [_token_rows(t, n) for t, n in ((y, "y"), (x, "x"), (out, "out"))]
    zp = _token_rows(z, "z") if z is not None else (None, 0, 0)
    if any(tuple(t.shape) != (b, hw, c) for t in (x, out) + ((z,) if z is not None else ())):
        raise RuntimeError("context_gate: y, x, z and out must have the same shape")
    ws = torch.empty(max(int(lib().sdetr_context_gate_workspace_floats(b, hw, c)), 4), device=y.device, dtype=torch.float32)
    rc = lib().sdetr_context_gate(*ops[0], *ops[1], *zp, b, hw, c, _req(w_mask, "w_mask", torch.float32),
                                  _req(b_mask, "b_mask", torch.float32), _req(w1, "w1", torch.float32), _req(w2, "w2", torch.float32),
                                  r, ws.data_ptr(), ws.numel(), *ops[2], _stream())
    _check(rc, "sdetr_context_gate")
    return out


def upsample_nearest_concat(hi, hi_hw, lo, lo_hw, out=None):
    """(b, Ho*Wo, 2C) = [nearest(hi) | lo]: hi (b, Hi*Wi, C), lo (b, Ho*Wo, C) views; torch's nearest index rule."""
    b, _, c = hi.shape
    ho, wo = lo_hw
    out = out if out is not None else torch.empty(b, ho * wo, 2 * c, device=hi.device, dtype=torch.float32)
    if tuple(lo.shape) != (b, ho * wo, c) or tuple(out.shape) != (b, ho * wo, 2 * c) or hi.shape[1] != hi_hw[0] * hi_hw[1]:
        raise RuntimeError("upsample_nearest_concat: shapes do not match")
    rc = lib().sdetr_upsample_nearest_concat(*_token_rows(hi, "hi"), int(hi_hw[0]), int(hi_hw[1]), *_token_rows(lo, "lo"), int(ho),
                                             int(wo), b, c, *_token_rows(out, "out"), _stream())
    _check(rc, "sdetr_upsample_nearest_concat")
    return out


def conv2d_f16x3_split_weight(w, groups: int, dgrad: bool = True):
    """(fwd_hi, fwd_lo, dgrad_hi, dgrad_lo, scale) of a (Cout, Cin / groups, k, k) fp32 weight in one pass: the pair for
    conv2d_f16x3 (Cout, k, k, Cin / groups) and, with ``dgrad``, the pair of the flipped, per-group transposed input-gradient
    weights (Cin, k, k, Cout / groups) (else None, None); scale: the power-of-two device scale of both (target 14)."""
    cout, cin_g, k, _ = w.shape
    scale = pow2_scale(w, 14)
    f_hi = torch.empty(cout, k, k, cin_g, device=w.device, dtype=torch.float16)
    f_lo = torch.empty_like(f_hi)
    d_hi = torch.empty(cin_g * groups, k, k, cout // groups, device=w.device, dtype=torch.float16) if dgrad else None
    d_lo = torch.empty_like(d_hi) if dgrad else None
    rc = lib().sdetr_conv2d_f16x3_split_weight(_req(w, "w", torch.float32), cout, cin_g * groups, int(groups), k, scale.data_ptr(),
                                               f_hi.data_ptr(), f_lo.data_ptr(), d_hi.data_ptr() if dgrad else None,
                                               d_lo.data_ptr() if dgrad else None, _stream())
    _check(rc, "sdetr_conv2d_f16x3_split_weight")
    return f_hi, f_lo, d_hi, d_lo, scale


def conv2d_f16x3_wgrad(dy, dy_scale, x, x_scale, hw, weight_shape, stride: int, cout_scale=None):
    """Weight gradient (Cout, Cin / groups, k, k) of y = conv(x, W): dy (b, Ho*Wo, Cout), x (b, H*W, Cin) views with unit channel
    stride, hw = (H, W); dy_scale / x_scale: their pow2_scale device scalars (target 12).  Bit-reproducible.
    cout_scale: optional (Cout,) fp32 factor per output channel, applied in the split sum's write."""
    b, _, cin = x.shape
    cout, cin_g, k, _ = (int(v) for v in weight_shape)
    groups = cin // cin_g
    pad = k // 2
    ho, wo = (hw[0] + 2 * pad - k) // stride + 1, (hw[1] + 2 * pad - k) // stride + 1
    if tuple(dy.shape) != (b, ho * wo, cout) or x.shape[1] != hw[0] * hw[1]:
        raise RuntimeError("conv2d_f16x3_wgrad: dy, x and the map size do not match")
    dw = torch.empty(cout, cin_g, k, k, device=x.device, dtype=torch.float32)
    ws = torch.empty(max(int(lib().sdetr_conv2d_f16x3_wgrad_workspace_floats(b, ho, wo, cin, cout, groups, k)), 4), device=x.device,
                     dtype=torch.float32)
    if cout_scale is not None and cout_scale.numel() != cout:
        raise RuntimeError(f"conv2d_f16x3_wgrad: cout_scale must have {cout} entries")
    cs = _req(cout_scale, "cout_scale", torch.float32) if cout_scale is not None else None
    rc = lib().sdetr_conv2d_f16x3_wgrad(*_token_rows(dy, "dy"), _req(dy_scale, "dy_scale", torch.float32), *_token_rows(x, "x"),
                                        _req(x_scale, "x_scale", torch.float32), b, int(hw[0]), int(hw[1]), cin, cout, groups, k,
                                        int(stride), cs, ws.data_ptr(), ws.numel(), dw.data_ptr(), _stream())
    _check(rc, "sdetr_conv2d_f16x3_wgrad")
    return dw


def conv2d_f16x3_dgrad(dy, dy_hw, a_scale, w_hi, w_lo, w_scale, groups: int, ksize: int, stride: int, hw, z=None, m=None, out=None):
    """Input gradient of a stride-1 or stride-2 convolution of an (H, W) = hw map with a fused epilogue:
    dx = conv^T(dy, W) (+ z), then 0 where m <= 0 (torch's threshold_backward(dx, m, 0)).  dy (b, Hy*Wy, Cout) view; W' = the
    (Cin, k, k, Cout / groups) input-gradient pair of conv2d_f16x3_split_weight; a_scale: pow2_scale of dy (target 12).
    z, m: optional (b, H*W, Cin) views, z may be ``out`` itself, m may not.  out: optional (b, H*W, Cin) view to write."""
    b, n, cin = dy.shape
    if n != dy_hw[0] * dy_hw[1]:
        raise RuntimeError(f"conv2d_f16x3_dgrad: dy has {n} rows per image, the map is {dy_hw[0]}x{dy_hw[1]}")
    cout = w_hi.shape[0]
    dx = out if out is not None else torch.empty(b, hw[0] * hw[1], cout, device=dy.device, dtype=torch.float32)
    for t, name in ((dx, "out"), (z, "z"), (m, "m")):
        if t is not None and tuple(t.shape) != (b, hw[0] * hw[1], cout):
            raise RuntimeError(f"conv2d_f16x3_dgrad: {name} must be ({b}, {hw[0] * hw[1]}, {cout})")
    zp = _token_rows(z, "z") if z is not None else (None, 0, 0)
    mp = _token_rows(m, "m") if m is not None else (None, 0, 0)
    rc = lib().sdetr_conv2d_f16x3_dgrad(*_token_rows(dy, "dy"), b, int(dy_hw[0]), int(dy_hw[1]), cin,
                                        _req(a_scale, "a_scale", torch.float32), _req(w_hi, "w_hi", torch.float16),
                                        _req(w_lo, "w_lo", torch.float16), _req(w_scale, "w_scale", torch.float32), *zp, *mp, cout,
                                        int(groups), int(ksize), int(stride), int(hw[0]), int(hw[1]), *_token_rows(dx, "dx"),
                                        _stream())
    _check(rc, "sdetr_conv2d_f16x3_dgrad")
    return dx


def frozen_bn_fold(w, bn, scale: bool = True, bias: bool = True):
    """(w * s, s, bias - running_mean * s) of a weight (Cout, ...) and a FrozenBatchNorm2d ``bn`` (s = weight * rsqrt(running_var
    + eps)), computed on the device in float64 and rounded to fp32 (sdetr_frozen_bn_fold), with no host read.
    s / the bias are None unless asked for."""
    cout = w.shape[0]
    wf = torch.empty(w.shape, device=w.device, dtype=torch.float32)
    s = torch.empty(cout, device=w.device, dtype=torch.float32) if scale else None
    bf = torch.empty(cout, device=w.device, dtype=torch.float32) if bias else None
    rc = lib().sdetr_frozen_bn_fold(_req(w, "w", torch.float32), cout, w.numel() // cout, _req(bn.weight, "bn.weight", torch.float32),
                                    _req(bn.bias, "bn.bias", torch.float32), _req(bn.running_mean, "bn.running_mean", torch.float32),
                                    _req(bn.running_var, "bn.running_var", torch.float32), float(bn.eps), wf.data_ptr(),
                                    s.data_ptr() if scale else None, bf.data_ptr() if bias else None, _stream())
    _check(rc, "sdetr_frozen_bn_fold")
    return wf, s, bf


def upsample_nearest_concat_backward(g_hi, lo_hw, hi_hw):
    """Gradient of hi in upsample_nearest_concat: g_hi (b, Ho*Wo, C) view (the first C channels of the concatenation's
    gradient) -> (b, Hi*Wi, C), each source pixel the fixed-order sum over the destination pixels that read it."""
    b, n, c = g_hi.shape
    if n != lo_hw[0] * lo_hw[1]:
        raise RuntimeError("upsample_nearest_concat_backward: shapes do not match")
    out = torch.empty(b, hi_hw[0] * hi_hw[1], c, device=g_hi.device, dtype=torch.float32)
    rc = lib().sdetr_upsample_nearest_concat_backward(*_token_rows(g_hi, "g"), int(lo_hw[0]), int(lo_hw[1]), int(hi_hw[0]),
                                                      int(hi_hw[1]), b, c, *_token_rows(out, "out"), _stream())
    _check(rc, "sdetr_upsample_nearest_concat_backward")
    return out


# ---- ChannelMapper in token layout (channel_mapper.ChannelMapper.forward_tokens) ----------------------------------------------
def _gn_rows(t, name, b, nv, c):
    if not (t.is_cuda and t.dtype == torch.float32 and tuple(t.shape) == (b, nv, c) and t.stride(2) == 1 and t.stride(1) == c):
        raise RuntimeError(f"{name} must be CUDA float32 ({b}, {nv}, {c}) with contiguous rows")
    if t.device.index != _current_device():
        raise RuntimeError(f"{name} lives on {t.device} but cuda:{_current_device()} is current")
    return t.stride(0) if b > 1 else nv * c


def group_norm_tokens_(tokens, level_sizes: Sequence[int], gamma, beta, num_groups: int, eps: float, out=None):
    """nn.GroupNorm of every level of ``tokens`` (b, Nv, C) in place, or into ``out`` (three launches for all levels).  ``tokens``
    may be a token-range view of a larger buffer (unit channel stride, rows C apart); ``out``, when given, has its image pitch;
    gamma / beta: (L, C) contiguous."""
    b, nv, c = tokens.shape
    L = len(level_sizes)
    pitch = _gn_rows(tokens, "group_norm_tokens_: tokens", b, nv, c)
    y = tokens if out is None else out
    if out is not None and _gn_rows(out, "group_norm_tokens_: out", b, nv, c) != pitch:
        raise RuntimeError("group_norm_tokens_: out must have the image pitch of tokens")
    if sum(level_sizes) != nv or tuple(gamma.shape) != (L, c) or tuple(beta.shape) != (L, c):
        raise RuntimeError(f"group_norm_tokens_: {nv} tokens, levels {list(level_sizes)}, gamma / beta must be ({L}, {c})")
    sizes = _host_i32(level_sizes)
    ws = torch.empty(max(int(lib().sdetr_group_norm_tokens_workspace_floats(b, c, int(num_groups), L, sizes)), 4),
                     device=tokens.device, dtype=torch.float32)
    rc = lib().sdetr_group_norm_tokens(tokens.data_ptr(), y.data_ptr(), pitch, b, c, L, sizes, _req(gamma, "gamma", torch.float32),
                                       _req(beta, "beta", torch.float32), int(num_groups), float(eps), ws.data_ptr(), ws.numel(),
                                       _stream())
    _check(rc, "sdetr_group_norm_tokens")
    return y


def group_norm_tokens_backward(dy, x, level_sizes: Sequence[int], gamma, num_groups: int, eps: float, dx=None,
                               dgamma: bool = True, dbeta: bool = True):
    """Gradient of group_norm_tokens_ -> (dx, dgamma, dbeta).  dy, x: (b, Nv, C) views with contiguous rows and one image pitch
    (x the forward's input); gamma: (L, C) contiguous.  ``dx``: optional destination with that pitch, may be ``x`` or ``dy``
    itself.  dgamma / dbeta: (L, C) tables when asked for, else None (and, with neither, one launch less)."""
    b, nv, c = x.shape
    L = len(level_sizes)
    pitch = _gn_rows(x, "group_norm_tokens_backward: x", b, nv, c)
    dx = dx if dx is not None else torch.empty(b, nv, c, device=x.device, dtype=torch.float32)
    if _gn_rows(dy, "group_norm_tokens_backward: dy", b, nv, c) != pitch or _gn_rows(dx, "group_norm_tokens_backward: dx", b, nv, c) != pitch:
        raise RuntimeError("group_norm_tokens_backward: dy, x and dx must have the same image pitch")
    if sum(level_sizes) != nv or tuple(gamma.shape) != (L, c):
        raise RuntimeError(f"group_norm_tokens_backward: {nv} tokens, levels {list(level_sizes)}, gamma must be ({L}, {c})")
    dg = torch.empty(L, c, device=x.device, dtype=torch.float32) if dgamma else None
    db = torch.empty(L, c, device=x.device, dtype=torch.float32) if dbeta else None
    sizes = _host_i32(level_sizes)
    ws = torch.empty(max(int(lib().sdetr_group_norm_tokens_backward_workspace_floats(b, c, int(num_groups), L, sizes)), 4),
                     device=x.device, dtype=torch.float32)
    rc = lib().sdetr_group_norm_tokens_backward(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), pitch, b, c, L, sizes,
                                                _req(gamma, "gamma", torch.float32), int(num_groups), float(eps),
                                                dg.data_ptr() if dg is not None else None, db.data_ptr() if db is not None else None,
                                                ws.data_ptr(), ws.numel(), _stream())
    _check(rc, "sdetr_group_norm_tokens_backward")
    return dx, dg, db


def token_lpos_keep(feat, pos, level_embeds, keep, level_sizes: Sequence[int], lpos=None):
    """feat / pos (b, Nv, C) tokens -> (lpos, x): lpos = pos + level_embeds[l], x = (feat + lpos) * keep, bit-identical to
    flatten_tokens[_pos] on the same values.  ``lpos``: optional destination, may be ``pos`` itself (in place)."""
    b, nv, c = feat.shape
    if tuple(pos.shape) != (b, nv, c) or sum(level_sizes) != nv or tuple(level_embeds.shape[1:]) != (c,):
        raise RuntimeError(f"token_lpos_keep: pos must be {(b, nv, c)}, the levels must sum to {nv}, level_embeds (L, {c})")
    lpos = lpos if lpos is not None else torch.empty_like(feat)
    x = torch.empty_like(feat)
    rc = lib().sdetr_token_lpos_keep(_req(feat, "feat", torch.float32), _req(pos, "pos", torch.float32),
                                     _req(level_embeds, "level_embeds", torch.float32), _req(keep, "keep", torch.float32),
                                     _host_i32(level_sizes), b, c, len(level_sizes), _req(lpos, "lpos", torch.float32), x.data_ptr(),
                                     _stream())
    _check(rc, "sdetr_token_lpos_keep")
    return lpos, x


# ---- detection loss (set_criterion.cu) ------------------------------------------------------------------------------------
SET_MAX_PROBLEMS = 128  # include/sdetr_b200.h SDETR_SET_MAX_PROBLEMS
SET_MAX_QUERIES = 4096  # SDETR_SET_MAX_QUERIES: the solver's shared-memory limit


class SetProblem(ctypes.Structure):
    """``sdetr_set_problem``: one (output, image) problem of the matcher / loss entry points."""
    _fields_ = [("logits", _vp), ("boxes", _vp), ("gt_boxes", _vp), ("gt_labels", _vp), ("src", _vp), ("tgt", _vp),
                ("grad_logits", _vp), ("grad_boxes", _vp), ("logit_stride", _i64), ("box_stride", _i64),
                ("num_queries", ctypes.c_int32), ("num_gt", ctypes.c_int32), ("num_pairs", ctypes.c_int32),
                ("output", ctypes.c_int32)]


def _problem_table(problems):
    if len(problems) > SET_MAX_PROBLEMS:
        raise RuntimeError(f"{len(problems)} (output, image) problems in one call; at most {SET_MAX_PROBLEMS}")
    return (SetProblem * max(len(problems), 1))(*problems)


def _num_boxes_args(num_boxes):
    """num_boxes: a Python number (host value) or a one-element float32 CUDA tensor (read by the kernels)."""
    if torch.is_tensor(num_boxes):
        if not (num_boxes.is_cuda and num_boxes.dtype == torch.float32 and num_boxes.numel() == 1):
            raise RuntimeError("num_boxes must be a number or a one-element CUDA float32 tensor")
        return 1.0, num_boxes.data_ptr()
    return float(num_boxes), None


def set_match(problems, num_classes: int, cost_class: float, cost_bbox: float, cost_giou: float, alpha: float, gamma: float,
              status):
    """Cost matrices + exact assignments of all ``problems`` (their src / tgt buffers are written) in one launch;
    status (len(problems),) int32 receives 1 for a problem with a non-finite cost.  -> the workspace holding every problem's
    (num_gt, num_queries) cost matrix, one after the other."""
    tab = _problem_table(problems)
    need = int(lib().sdetr_set_match_workspace_floats(tab, len(problems)))
    ws = torch.empty(max(need, 1), device=status.device, dtype=torch.float32)
    _check(lib().sdetr_set_match(tab, len(problems), int(num_classes), float(cost_class), float(cost_bbox), float(cost_giou),
                                 float(alpha), float(gamma), _req(status, "status", torch.int32), ws.data_ptr(), ws.numel(),
                                 _stream()), "sdetr_set_match")
    return ws


def set_assign(problems, cost, status):
    """Exact assignments of given costs: ``cost`` holds every problem's (num_gt, num_queries) fp32 matrix, one after the other."""
    tab = _problem_table(problems)
    _check(lib().sdetr_set_assign(tab, len(problems), _req(cost, "cost", torch.float32), cost.numel(),
                                  _req(status, "status", torch.int32), _stream()), "sdetr_set_assign")


def set_loss_forward(problems, num_outputs: int, num_classes: int, alpha: float, gamma: float, status, num_boxes, loss):
    """Writes loss (num_outputs, 3) float32, contiguous: (loss_class, loss_bbox, loss_giou) per output."""
    tab = _problem_table(problems)
    need = int(lib().sdetr_set_loss_workspace_floats(tab, len(problems)))
    ws = torch.empty(max(need, 1), device=loss.device, dtype=torch.float32)
    nb_host, nb_dev = _num_boxes_args(num_boxes)
    _check(lib().sdetr_set_loss_forward(tab, len(problems), int(num_outputs), int(num_classes), float(alpha), float(gamma),
                                        status.data_ptr() if status is not None else None, nb_host, nb_dev, ws.data_ptr(),
                                        ws.numel(), _req(loss, "loss", torch.float32), _stream()), "sdetr_set_loss_forward")
    return loss


def set_loss_backward(problems, num_outputs: int, num_classes: int, alpha: float, gamma: float, status, num_boxes, grad_loss):
    """Writes every problem's grad_logits / grad_boxes for the (num_outputs, 3) upstream gradient ``grad_loss``."""
    tab = _problem_table(problems)
    nb_host, nb_dev = _num_boxes_args(num_boxes)
    _check(lib().sdetr_set_loss_backward(tab, len(problems), int(num_outputs), int(num_classes), float(alpha), float(gamma),
                                         status.data_ptr() if status is not None else None, nb_host, nb_dev,
                                         _req(grad_loss, "grad_loss", torch.float32), _stream()), "sdetr_set_loss_backward")


# ---- contrastive denoising queries (denoising.cu) -----------------------------------------------------------------------------
CDN_MAX_IMAGES = 128  # include/sdetr_b200.h SDETR_CDN_MAX_IMAGES


class CDNImage(ctypes.Structure):
    """``sdetr_cdn_image``: one image's gts for the denoising-query entry points."""
    _fields_ = [("gt_labels", _vp), ("gt_boxes", _vp), ("num_gt", ctypes.c_int32), ("reserved", ctypes.c_int32)]


def _opt(t, name, dtype):
    return _req(t, name, dtype) if t is not None else None


def cdn_queries(labels, boxes, draws, weight, num_classes: int, embed_dim: int, label_threshold: float, box_noise_scale: float,
                num_queries: int, groups: int, max_gt: int):
    """labels / boxes: per-image int64 (n_i,) / float32 (n_i, 4) contiguous CUDA tensors; draws: (label_rand, label_randint,
    box_randint, box_rand), None where that noise is off.  -> (label_queries (b, D, C), box_queries (b, D, 4), noised_labels
    (b, D) int32, attn_mask (T, T) bool, status (b,) int32) with D = 2 * groups * max_gt, T = D + num_queries."""
    b = len(labels)
    if b > CDN_MAX_IMAGES:
        raise RuntimeError(f"{b} images in one call; at most {CDN_MAX_IMAGES}")
    K, C = int(num_classes), int(embed_dim)
    dev = weight.device
    D = 2 * groups * max_gt
    ims = (CDNImage * max(b, 1))(*[CDNImage(gt_labels=_req(lb, "gt_labels", torch.int64) if lb.numel() else None,
                                            gt_boxes=_req(bx, "gt_boxes", torch.float32) if lb.numel() else None,
                                            num_gt=lb.numel()) for lb, bx in zip(labels, boxes)])
    label_q = torch.empty(b, D, C, device=dev, dtype=torch.float32)
    box_q = torch.empty(b, D, 4, device=dev, dtype=torch.float32)
    noised = torch.empty(b, D, device=dev, dtype=torch.int32)
    mask = torch.empty(D + num_queries, D + num_queries, device=dev, dtype=torch.bool)
    status = torch.empty(b, device=dev, dtype=torch.int32)
    lr, li, bs, br = draws
    _check(lib().sdetr_cdn_queries(ims, b, _opt(lr, "label_rand", torch.float32), _opt(li, "label_randint", torch.int64),
                                   _opt(bs, "box_randint", torch.float32), _opt(br, "box_rand", torch.float32),
                                   float(label_threshold), float(box_noise_scale), _req(weight, "weight", torch.float32), K, C,
                                   *[int(x) for x in weight.shape],
                                   int(num_queries), int(groups), int(max_gt), label_q.data_ptr(), box_q.data_ptr(),
                                   noised.data_ptr(), mask.data_ptr(), status.data_ptr(), _stream()), "sdetr_cdn_queries")
    return label_q, box_q, noised, mask, status


def cdn_queries_backward(grad_label_queries, noised_labels, num_classes: int):
    """(b, D, C) gradient of the label queries + the forward's noised labels -> grad of label_encoder.weight (K, C)."""
    C = grad_label_queries.shape[-1]
    gw = torch.empty(num_classes, C, device=grad_label_queries.device, dtype=torch.float32)
    _check(lib().sdetr_cdn_queries_backward(_req(grad_label_queries, "grad_label_queries", torch.float32),
                                            _req(noised_labels, "noised_labels", torch.int32), noised_labels.numel(),
                                            int(num_classes), C, gw.data_ptr(), _stream()), "sdetr_cdn_queries_backward")
    return gw


def cdn_loss_indices(counts: Sequence[int], groups: int, max_gt: int, device):
    """-> (2, groups * sum(counts)) int64: per image the (g * max_gt + t, t) pairs of compute_dn_loss, image after image."""
    if len(counts) > CDN_MAX_IMAGES:
        raise RuntimeError(f"{len(counts)} images in one call; at most {CDN_MAX_IMAGES}")
    out = torch.empty(2, groups * sum(counts), device=device, dtype=torch.int64)
    _check(lib().sdetr_cdn_loss_indices(_host_i32(counts) if counts else None, len(counts), int(groups), int(max_gt),
                                        out.data_ptr() if out.numel() else None, _stream()), "sdetr_cdn_loss_indices")
    return out


# ---- detection post-processing (postprocess.cu) -------------------------------------------------------------------------------
POSTPROCESS_MAX_K = 4096  # include/sdetr_b200.h SDETR_POSTPROCESS_MAX_K
_SIZES_DTYPES = {torch.int64: 0, torch.int32: 1, torch.float32: 2}  # SDETR_SIZES_*


def _strided(t, name, dtype):
    """The checks of _req but for a unit last stride instead of contiguity (a copy when the last stride is not 1)."""
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.stride(-1) != 1:
        t = t.contiguous()
    _req(t.as_strided((1,), (1,)) if t.numel() else t, name, dtype)  # device and dtype, on a one-element view
    return t


def postprocess(logits, boxes, target_sizes, k: int, confidence_score: float, iou_threshold: float):
    """logits (b, Q, K) fp32 and boxes (b, Q, 4) cxcywh fp32 with any batch / query strides, target_sizes (b, 2) (h, w) int64,
    int32 or float32 -> (scores (b, k) fp32, labels (b, k) int64, boxes (b, k, 4) fp32, count (b,) int32 or None).  A threshold
    > 0 turns its filter on; then the first count[i] entries of row i are its kept ones, else count is None."""
    logits = _strided(logits, "pred_logits", torch.float32)
    boxes = _strided(boxes, "pred_boxes", torch.float32)
    if target_sizes.dtype not in _SIZES_DTYPES:
        raise RuntimeError(f"target_sizes must be int64, int32 or float32, got {target_sizes.dtype}")
    sizes = _strided(target_sizes, "target_sizes", target_sizes.dtype).contiguous()
    b, Q, K = logits.shape
    if tuple(boxes.shape) != (b, Q, 4):
        raise RuntimeError(f"pred_boxes must be ({b}, {Q}, 4), got {tuple(boxes.shape)}")
    if not 0 <= k <= Q * K:
        raise RuntimeError(f"selected index k out of range: k={k}, {Q * K} scores per image")
    if k > POSTPROCESS_MAX_K:
        raise RuntimeError(f"k={k}: the post-processing kernel selects at most {POSTPROCESS_MAX_K} boxes per image")
    filters = confidence_score > 0 or iou_threshold > 0
    dev = logits.device
    scores = torch.empty(b, k, device=dev, dtype=torch.float32)
    labels = torch.empty(b, k, device=dev, dtype=torch.int64)
    out_boxes = torch.empty(b, k, 4, device=dev, dtype=torch.float32)
    count = torch.empty(b, device=dev, dtype=torch.int32) if filters else None
    if b == 0 or k == 0:  # nothing to select (torch.topk with k = 0 returns empty rows)
        if count is not None:
            count.zero_()
        return scores, labels, out_boxes, count
    ws = torch.empty(lib().sdetr_postprocess_workspace(b, Q, K), device=dev, dtype=torch.uint8)
    _check(lib().sdetr_postprocess(logits.data_ptr(), logits.stride(0), logits.stride(1), boxes.data_ptr(), boxes.stride(0),
                                   boxes.stride(1), sizes.data_ptr(), _SIZES_DTYPES[sizes.dtype], b, Q, K, int(k),
                                   float(confidence_score), float(iou_threshold), scores.data_ptr(), labels.data_ptr(),
                                   out_boxes.data_ptr(), count.data_ptr() if count is not None else None, ws.data_ptr(),
                                   ws.numel(), _stream()), "sdetr_postprocess")
    return scores, labels, out_boxes, count


# ---- ResNet backbone in token layout (backbone.ResNetBackbone.forward_tokens) ------------------------------------------------
def resnet_stem(x, weight, bias):
    """ReLU(conv 7x7 / 2, padding 3 (x) + bias) -> (b, Ho*Wo, 64) token rows.  x: (b, 3, H, W) NCHW contiguous fp32 CUDA;
    weight: (147, 64) = the folded (64, 3, 7, 7) weight as W.reshape(64, 147).T, contiguous; bias (64)."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.is_contiguous()):
        raise RuntimeError("resnet_stem: x must be a contiguous CUDA float32 (b, 3, H, W) tensor")
    b, _, H, W = x.shape
    if tuple(weight.shape) != (147, 64) or tuple(bias.shape) != (64,):
        raise RuntimeError("resnet_stem: weight must be (147, 64) and bias (64)")
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty(b, ho * wo, 64, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_resnet_stem(_req(x, "x", torch.float32), b, H, W, _req(weight, "weight", torch.float32),
                                 _req(bias, "bias", torch.float32), y.data_ptr(), _stream())
    _check(rc, "sdetr_resnet_stem")
    return y


def maxpool3x3s2_tokens(x, hw, out=None):
    """3x3 / stride 2 / padding 1 max-pool (torch's max_pool2d) of (b, H*W, C) token rows, hw = (H, W) -> (b, Ho*Wo, C)."""
    b, n, c = x.shape
    H, W = hw
    if n != H * W:
        raise RuntimeError(f"maxpool3x3s2_tokens: x has {n} rows per image, the map is {H}x{W}")
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = out if out is not None else torch.empty(b, ho * wo, c, device=x.device, dtype=torch.float32)
    if tuple(y.shape) != (b, ho * wo, c):
        raise RuntimeError(f"maxpool3x3s2_tokens: out must be ({b}, {ho * wo}, {c})")
    rc = lib().sdetr_maxpool3x3s2_tokens(*_token_rows(x, "x"), b, int(H), int(W), c, *_token_rows(y, "out"), _stream())
    _check(rc, "sdetr_maxpool3x3s2_tokens")
    return y


# ---- ConvNeXt backbone in token layout (convnext.ConvNeXtBackbone.forward_tokens) ----------------------------------------------
ACT_GELU = 2  # gemm_f16x3_ex: exact GELU applied to the input as it loads


def gemm_f16x3_ex(x, a_scale, w_hi, w_lo, w_scale, bias=None, act=0, col_scale=None, z=None, out=None):
    """out = z + col_scale * (act(x) @ W.T + bias) on the projection GEMM (3xFP16, device scales, no host synchronisation).
    x (..., K) fp32 with unit last stride and rows of a 16-byte multiple; a_scale: pow2_scale of x (target 12); (w_hi, w_lo,
    w_scale): split_f16_pair_dev of W (N, K); act 0 none, 1 ReLU, 2 exact GELU on x as it loads; col_scale (N) or None; z: a
    (..., N) tensor of x's leading shape with unit last stride, or None; out: None (a fresh tensor) or such a tensor, which may be
    z itself."""
    K = x.shape[-1]
    N = w_hi.shape[0]
    if not (x.is_cuda and x.dtype == torch.float32 and x.stride(-1) == 1):
        raise RuntimeError("gemm_f16x3_ex needs a CUDA float32 input with unit last stride")
    x2 = x if x.dim() == 2 else x.reshape(-1, K)
    M = x2.shape[0]
    lead = tuple(x.shape[:-1])

    def rows(t, name):
        if not (t.is_cuda and t.dtype == torch.float32 and tuple(t.shape) == lead + (N,) and t.stride(-1) == 1):
            raise RuntimeError(f"gemm_f16x3_ex: {name} must be a CUDA float32 {lead + (N,)} tensor with unit last stride")
        t2 = t if t.dim() == 2 else t.view(-1, N)
        return t2, (t2.stride(0) if M > 1 else N)

    y = out if out is not None else torch.empty(*lead, N, device=x.device, dtype=torch.float32)
    y2, ldc = rows(y, "out")
    zp, ldz = (None, 0)
    if z is not None:
        z2, ldz = rows(z, "z")
        zp = z2.data_ptr()
    if col_scale is not None and tuple(col_scale.shape) != (N,):
        raise RuntimeError(f"gemm_f16x3_ex: col_scale must be ({N},)")
    rc = lib().sdetr_gemm_f16x3_ex(x2.data_ptr(), x2.stride(0) if M > 1 else K, _req(a_scale, "a_scale", torch.float32),
                                   _req(w_hi, "w_hi", torch.float16), _req(w_lo, "w_lo", torch.float16),
                                   _req(w_scale, "w_scale", torch.float32),
                                   _req(bias, "bias", torch.float32) if bias is not None else None,
                                   _req(col_scale, "col_scale", torch.float32) if col_scale is not None else None, zp, ldz,
                                   y2.data_ptr(), ldc, M, N, K, int(act), _stream())
    _check(rc, "sdetr_gemm_f16x3_ex")
    return y


def convnext_stem(x, weight, bias, ln_weight, ln_bias, eps: float = 1e-6):
    """LayerNorm(conv 4x4 / 4 (x) + bias) over C -> (b, (H // 4) * (W // 4), C) token rows.  x: (b, 3, H, W) NCHW contiguous fp32
    CUDA; weight: (48, C) = W.reshape(C, 48).T, contiguous; bias, ln_weight, ln_bias (C)."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.is_contiguous()):
        raise RuntimeError("convnext_stem: x must be a contiguous CUDA float32 (b, 3, H, W) tensor")
    b, _, H, W = x.shape
    C = weight.shape[1]
    if weight.dim() != 2 or weight.shape[0] != 48 or any(tuple(t.shape) != (C,) for t in (bias, ln_weight, ln_bias)):
        raise RuntimeError("convnext_stem: weight must be (48, C) and bias, ln_weight, ln_bias (C)")
    y = torch.empty(b, (H // 4) * (W // 4), C, device=x.device, dtype=torch.float32)
    if y.numel() == 0:  # an image under 4 pixels high or wide: no output pixel
        return y
    rc = lib().sdetr_convnext_stem(_req(x, "x", torch.float32), b, H, W, C, _req(weight, "weight", torch.float32),
                                   _req(bias, "bias", torch.float32), _req(ln_weight, "ln_weight", torch.float32),
                                   _req(ln_bias, "ln_bias", torch.float32), float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_convnext_stem")
    return y


def dwconv7x7_layernorm_tokens(x, hw, weight, bias, ln_weight, ln_bias, eps: float = 1e-6):
    """LayerNorm(depthwise conv 7x7, padding 3 (x) + bias) over C of (b, H*W, C) contiguous token rows, hw = (H, W) -> a new
    (b, H*W, C) tensor.  weight: (49, C) = W.reshape(C, 49).T, contiguous."""
    b, n, C = x.shape
    H, W = hw
    if n != H * W:
        raise RuntimeError(f"dwconv7x7_layernorm_tokens: x has {n} rows per image, the map is {H}x{W}")
    if tuple(weight.shape) != (49, C) or any(tuple(t.shape) != (C,) for t in (bias, ln_weight, ln_bias)):
        raise RuntimeError("dwconv7x7_layernorm_tokens: weight must be (49, C) and bias, ln_weight, ln_bias (C)")
    y = torch.empty_like(x)
    rc = lib().sdetr_dwconv7x7_layernorm_tokens(_req(x, "x", torch.float32), b, int(H), int(W), C,
                                                _req(weight, "weight", torch.float32), _req(bias, "bias", torch.float32),
                                                _req(ln_weight, "ln_weight", torch.float32), _req(ln_bias, "ln_bias", torch.float32),
                                                float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_dwconv7x7_layernorm_tokens")
    return y


def layernorm_tokens_s2d(x, hw, ln_weight, ln_bias, eps: float = 1e-6):
    """LayerNorm over C of (b, H*W, C) contiguous token rows, written space-to-depth -> (b, (H // 2) * (W // 2), 4 C) with row
    (y, x) holding the normalised pixel (2 y + dy, 2 x + dx) at columns (2 dy + dx) * C + c."""
    b, n, C = x.shape
    H, W = hw
    if n != H * W:
        raise RuntimeError(f"layernorm_tokens_s2d: x has {n} rows per image, the map is {H}x{W}")
    if any(tuple(t.shape) != (C,) for t in (ln_weight, ln_bias)):
        raise RuntimeError("layernorm_tokens_s2d: ln_weight and ln_bias must be (C)")
    y = torch.empty(b, (H // 2) * (W // 2), 4 * C, device=x.device, dtype=torch.float32)
    if y.numel() == 0:  # a map of one row or column: no output pixel
        return y
    rc = lib().sdetr_layernorm_tokens_s2d(_req(x, "x", torch.float32), b, int(H), int(W), C,
                                          _req(ln_weight, "ln_weight", torch.float32), _req(ln_bias, "ln_bias", torch.float32),
                                          float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_layernorm_tokens_s2d")
    return y


# ---- Swin Transformer backbone in token layout (swin.SwinTransformerBackbone.forward_tokens) -------------------------------
def window_attention_tokens(qkv, hw, qkv_bias, rel_bias, num_heads: int, window, shift):
    """Shifted-window multi-head attention of V1 Swin from the QKV Linear's output: qkv (b, H*W, 3C) contiguous token rows in
    raster order, hw = (H, W), qkv_bias (3C), rel_bias (num_heads, N, N) the expanded relative position bias (N = window[0] *
    window[1]), window and shift the block's (h, w) window and nominal shift -> a new (b, H*W, C) tensor, the attention output
    before the projection at each pixel.  Padding, roll and the shift mask follow the reference (see sdetr_b200.h)."""
    b, n, c3 = qkv.shape
    H, W = hw
    C = c3 // 3
    if n != H * W or c3 != 3 * C:
        raise RuntimeError(f"window_attention_tokens: qkv must be (b, {H * W}, 3C), got {tuple(qkv.shape)}")
    N = int(window[0]) * int(window[1])
    if tuple(qkv_bias.shape) != (3 * C,) or tuple(rel_bias.shape) != (num_heads, N, N):
        raise RuntimeError(f"window_attention_tokens: qkv_bias must be ({3 * C},) and rel_bias ({num_heads}, {N}, {N})")
    y = torch.empty(b, n, C, device=qkv.device, dtype=torch.float32)
    rc = lib().sdetr_window_attention_tokens(_req(qkv, "qkv", torch.float32), _req(qkv_bias, "qkv_bias", torch.float32),
                                             _req(rel_bias, "rel_bias", torch.float32), b, int(H), int(W), C, int(num_heads),
                                             int(window[0]), int(window[1]), int(shift[0]), int(shift[1]), y.data_ptr(), _stream())
    _check(rc, "sdetr_window_attention_tokens")
    return y


def patch_merge_layernorm_tokens(x, hw, ln_weight, ln_bias, eps: float = 1e-5):
    """PatchMerging's pad, 2x2 concatenation and LayerNorm over 4C: x (b, H*W, C) contiguous token rows, hw = (H, W) -> a new
    (b, ceil(H / 2) * ceil(W / 2), 4C) tensor, row (y, x) holding pixel (2y + dy, 2x + dx) at columns (2 dx + dy) * C + c."""
    b, n, C = x.shape
    H, W = hw
    if n != H * W:
        raise RuntimeError(f"patch_merge_layernorm_tokens: x has {n} rows per image, the map is {H}x{W}")
    if any(tuple(t.shape) != (4 * C,) for t in (ln_weight, ln_bias)):
        raise RuntimeError(f"patch_merge_layernorm_tokens: ln_weight and ln_bias must be ({4 * C},)")
    y = torch.empty(b, ((H + 1) // 2) * ((W + 1) // 2), 4 * C, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_patch_merge_layernorm_tokens(_req(x, "x", torch.float32), b, int(H), int(W), C,
                                                  _req(ln_weight, "ln_weight", torch.float32),
                                                  _req(ln_bias, "ln_bias", torch.float32), float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_patch_merge_layernorm_tokens")
    return y


def layernorm_tokens(x, ln_weight, ln_bias, eps: float = 1e-5):
    """LayerNorm over the last dimension C (a multiple of 64 up to 1536) of contiguous fp32 rows -> a new tensor of x's shape."""
    C = x.shape[-1]
    if any(tuple(t.shape) != (C,) for t in (ln_weight, ln_bias)):
        raise RuntimeError(f"layernorm_tokens: ln_weight and ln_bias must be ({C},)")
    y = torch.empty_like(x, memory_format=torch.contiguous_format)
    rc = lib().sdetr_layernorm_tokens(_req(x, "x", torch.float32), x.numel() // C if C else 0, C,
                                      _req(ln_weight, "ln_weight", torch.float32), _req(ln_bias, "ln_bias", torch.float32),
                                      float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_layernorm_tokens")
    return y


# ---- FocalNet backbone in token layout (focalnet.FocalNetBackbone.forward_tokens) -------------------------------------------
def focalnet_stem(x, weight, bias, ln_weight, ln_bias, eps: float = 1e-5):
    """LayerNorm(conv 7x7 / 4, padding 2 (x) + bias) over C on the image zero-padded to a multiple of 4 -> (b, ceil(H / 4) *
    ceil(W / 4), C) token rows.  x: (b, 3, H, W) NCHW contiguous fp32 CUDA; weight: (147, C) = W.reshape(C, 147).T, contiguous;
    bias, ln_weight, ln_bias (C)."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3 and x.is_contiguous()):
        raise RuntimeError("focalnet_stem: x must be a contiguous CUDA float32 (b, 3, H, W) tensor")
    b, _, H, W = x.shape
    C = weight.shape[1]
    if weight.dim() != 2 or weight.shape[0] != 147 or any(tuple(t.shape) != (C,) for t in (bias, ln_weight, ln_bias)):
        raise RuntimeError("focalnet_stem: weight must be (147, C) and bias, ln_weight, ln_bias (C)")
    y = torch.empty(b, ((H + 3) // 4) * ((W + 3) // 4), C, device=x.device, dtype=torch.float32)
    rc = lib().sdetr_focalnet_stem(_req(x, "x", torch.float32), b, H, W, C, _req(weight, "weight", torch.float32),
                                   _req(bias, "bias", torch.float32), _req(ln_weight, "ln_weight", torch.float32),
                                   _req(ln_bias, "ln_bias", torch.float32), float(eps), y.data_ptr(), _stream())
    _check(rc, "sdetr_focalnet_stem")
    return y


def focal_context_partials(b: int, hw, C: int, device):
    """the workspace of the last focal level's partial channel sums (focal_level_tokens / focal_global_context)"""
    n = int(lib().sdetr_focal_context_workspace_floats(b, int(hw[0]), int(hw[1]), C))
    return torch.empty(max(n, 4), device=device, dtype=torch.float32)


def _rows_view(t, name, b, n, c):
    """(pointer, row stride) of a (b, n, c) fp32 CUDA view whose rows are one stride apart (a column slice of a contiguous
    tensor) with unit channel stride"""
    if not (t.is_cuda and t.dtype == torch.float32 and tuple(t.shape) == (b, n, c) and t.stride(2) == 1
            and (b * n <= 1 or t.stride(0) == n * t.stride(1))):
        raise RuntimeError(f"{name} must be a CUDA float32 ({b}, {n}, {c}) view with rows one stride apart and unit channel stride")
    if t.device.index != _current_device():
        raise RuntimeError(f"{name} lives on {t.device} but cuda:{_current_device()} is current")
    return t.data_ptr(), (t.stride(1) if n > 1 else t.stride(0) if b > 1 else c)


def focal_level_tokens(ctx, gate, hw, weight, ctx_all, first: bool, out=True, partials=None):
    """One focal level: p = GELU(depthwise conv k x k, padding k // 2 (ctx)), ctx_all = (0 if first else ctx_all) + p * gate.
    ctx: (b, H*W, C) view with rows one stride apart (e.g. a column slice of f's output); gate: (b, H*W, 1) view likewise;
    weight: (k * k, C) = W.reshape(C, k * k).T, contiguous; ctx_all: contiguous (b, H*W, C), updated in place.  out: True (a new
    tensor receives p, returned), or False (p not written, None returned); partials: None, or on the last level the workspace
    of focal_context_partials, which receives its per-tile channel sums."""
    b, n, C = ctx.shape
    H, W = hw
    if n != H * W:
        raise RuntimeError(f"focal_level_tokens: ctx has {n} rows per image, the map is {H}x{W}")
    kk = weight.shape[0]
    k = int(round(kk ** 0.5))
    if weight.dim() != 2 or k * k != kk or weight.shape[1] != C:
        raise RuntimeError(f"focal_level_tokens: weight must be (k * k, {C})")
    cp, ldc = _rows_view(ctx, "ctx", b, n, C)
    gp, ldg = _rows_view(gate, "gate", b, n, 1)
    if not (ctx_all.is_cuda and tuple(ctx_all.shape) == (b, n, C) and ctx_all.is_contiguous()):
        raise RuntimeError(f"focal_level_tokens: ctx_all must be a contiguous ({b}, {n}, {C}) tensor")
    y = torch.empty(b, n, C, device=ctx.device, dtype=torch.float32) if out else None
    rc = lib().sdetr_focal_level_tokens(cp, ldc, gp, ldg, _req(weight, "weight", torch.float32), k, b, int(H), int(W), C,
                                        int(bool(first)), y.data_ptr() if y is not None else None,
                                        _req(ctx_all, "ctx_all", torch.float32),
                                        _req(partials, "partials", torch.float32) if partials is not None else None,
                                        partials.numel() if partials is not None else 0, _stream())
    _check(rc, "sdetr_focal_level_tokens")
    return y


def focal_global_context(partials, gate, hw, ctx_all, focal_level: int, normalize: bool):
    """ctx_all = (ctx_all + GELU(mean over each image's pixels of ctx_L) * gate) [/ (focal_level + 1)] in place, the mean from the
    last focal level's partials.  gate: (b, H*W, 1) view with rows one stride apart."""
    b, n, C = ctx_all.shape
    H, W = hw
    if n != H * W or not ctx_all.is_contiguous():
        raise RuntimeError(f"focal_global_context: ctx_all must be a contiguous (b, {H * W}, C) tensor")
    gp, ldg = _rows_view(gate, "gate", b, n, 1)
    rc = lib().sdetr_focal_global_context(_req(partials, "partials", torch.float32), partials.numel(), gp, ldg, b, int(H), int(W), C,
                                          int(focal_level), int(bool(normalize)), _req(ctx_all, "ctx_all", torch.float32), _stream())
    _check(rc, "sdetr_focal_global_context")
    return ctx_all


def focal_modulate(q, h, out=None):
    """out = q * h: q (b, n, C) view with rows one stride apart (f's output's first C columns), h contiguous (b, n, C); out
    None (a new tensor) or a contiguous (b, n, C) tensor, which may be h."""
    b, n, C = h.shape
    qp, ldq = _rows_view(q, "q", b, n, C)
    y = out if out is not None else torch.empty_like(h)
    if tuple(y.shape) != (b, n, C) or not y.is_contiguous():
        raise RuntimeError(f"focal_modulate: out must be a contiguous ({b}, {n}, {C}) tensor")
    rc = lib().sdetr_focal_modulate(qp, ldq, _req(h, "h", torch.float32), b * n, C, y.data_ptr(), _stream())
    _check(rc, "sdetr_focal_modulate")
    return y


def layernorm_scale_add_tokens_(t, y, ln_weight, ln_bias, gamma, eps: float = 1e-5):
    """t = t + gamma * LayerNorm(y) over the last dimension C (a multiple of 64 up to 1536), in place; t and y contiguous of the
    same shape; returns t"""
    C = y.shape[-1]
    if tuple(t.shape) != tuple(y.shape) or any(tuple(v.shape) != (C,) for v in (ln_weight, ln_bias, gamma)):
        raise RuntimeError(f"layernorm_scale_add_tokens_: t must have y's shape and ln_weight, ln_bias, gamma ({C},)")
    rc = lib().sdetr_layernorm_scale_add_tokens(_req(y, "y", torch.float32), y.numel() // C if C else 0, C,
                                                _req(ln_weight, "ln_weight", torch.float32), _req(ln_bias, "ln_bias", torch.float32),
                                                float(eps), _req(gamma, "gamma", torch.float32), _req(t, "t", torch.float32),
                                                _stream())
    _check(rc, "sdetr_layernorm_scale_add_tokens")
    return t
