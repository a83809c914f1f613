"""Debug aid: install() wraps the C-ABI wrappers / GEMM entry points so that the first call producing a non-finite
output from finite inputs is reported (used with SDETR_POISON / SDETR_TRACE_NAN, see tests/conftest.py)."""
import torch
import torch.nn.functional as F

COUNT = [0]
FOUND = [False]


def finite(x):
    outs = x if isinstance(x, (tuple, list)) else (x,)
    for t in outs:
        if torch.is_tensor(t) and t.is_cuda and t.is_floating_point() and t.numel() and not bool(torch.isfinite(t).all()):
            return False
    return True


def _wrap(mod, name):
    fn = getattr(mod, name)

    def inner(*a, **kw):
        tens = [t for t in list(a) + list(kw.values()) if torch.is_tensor(t)]
        fin_in = finite(tens)
        out = fn(*a, **kw)
        COUNT[0] += 1
        res = out if out is not None else a[0]
        if not FOUND[0] and not finite(res):
            from salience_detr_b200 import gemm
            shapes = [(tuple(t.shape), str(t.dtype)[6:], t.is_contiguous(), tuple(t.stride())) for t in tens]
            print("\n[nan_trace] call #%d %s (gemm.MODE=%s): non-finite output, inputs finite: %s\n    %s" % (COUNT[0], name, gemm.MODE, fin_in, shapes), flush=True)
            outs = res if isinstance(res, (tuple, list)) else (res,)
            for i, t in enumerate(outs):
                if torch.is_tensor(t) and t.is_floating_point():
                    bad = (~torch.isfinite(t)).nonzero()
                    if bad.numel():
                        print("    out[%d] shape %s stride %s: %d bad, first %s last %s" % (i, tuple(t.shape), tuple(t.stride()), bad.shape[0], bad[0].tolist(), bad[-1].tolist()), flush=True)
            if fin_in:
                FOUND[0] = True
        return out
    setattr(mod, name, inner)


def install():
    from salience_detr_b200 import cabi, gemm
    for name in ("token_gather", "class_max_times_fg", "topk_desc", "rows_gather_add", "add_layernorm", "rows_scatter_",
                 "token_scatter_", "background_embed_", "msda_fused_forward", "salience_select", "order_prefixes",
                 "flatten_tokens", "zero_masked_rows_", "score_modulate_", "split_tf32",
                 "gemm_3xtf32_raw", "gemm_3xtf32"):
        if hasattr(cabi, name):
            _wrap(cabi, name)
    _wrap(gemm, "linear")
    _wrap(F, "linear")
    _wrap(F, "scaled_dot_product_attention")
    _wrap(F, "layer_norm")
