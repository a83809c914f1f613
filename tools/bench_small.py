"""Latency of the small (launch-bound) pieces with a warm L2, as they run inside a step: small-M dense projections
(hand-written wgmma kernel vs cuBLAS fp32) and the 300-token pre-attention (fused kernels vs library path)."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import salience_detr_b200 as pkg
import salience_detr_b200.salience_transformer as st
from salience_detr_b200.synthetic import build_model

dev = "cuda:0"


def timeit(fn, reps=30):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b) * 1000)
    return statistics.median(ts)


def graph_time(fn, reps=20, inner=20):
    """Per-call time inside a CUDA graph (no launch gaps from Python)."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(inner):
                fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s); g.replay(); b.record(s); s.synchronize(); ts.append(a.elapsed_time(b) * 1000 / inner)
    return statistics.median(ts)


print("small dense projections, per call inside a CUDA graph (us): own wgmma kernel | cuBLAS fp32")
for name, M, K, N, act in [("mask l3 fc1", 546, 256, 256, None), ("mask l3 fc2", 546, 256, 128, None), ("mask l3 fc3", 546, 128, 64, "gelu"),
                           ("mask l3 fc4", 546, 64, 1, "gelu"), ("mask l2 fc1", 2100, 256, 256, None), ("mask l2 fc3", 2100, 128, 64, "gelu"),
                           ("mask l1 fc1", 8400, 256, 256, None), ("mask l1 fc2", 8400, 256, 128, None), ("mask l1 fc3", 8400, 128, 64, "gelu"),
                           ("mask l1 fc4", 8400, 64, 1, "gelu"), ("mask l0 fc3", 33600, 128, 64, "gelu"), ("mask l0 fc4", 33600, 64, 1, "gelu"),
                           ("class L5", 4544, 256, 91, None), ("proj L5", 4544, 256, 384, None), ("class L0", 22726, 256, 91, None)]:
    x = torch.randn(M, K, device=dev); w = torch.randn(N, K, device=dev) / K ** 0.5; b = torch.randn(N, device=dev)
    r = []
    for mode in ("tcgen05", "fp32"):
        pkg.gemm.MODE = mode
        r.append(graph_time(lambda: pkg.gemm.linear(x, w, b, input_act=act)))
    print(f"  {name:12s} M={M:6d} K={K:4d} N={N:4d} | {r[0]:7.1f} | {r[1]:7.1f}")
pkg.gemm.MODE = "auto"

model = build_model().to(dev)
layer = model.encoder.layers[0]
torch.manual_seed(0)
for b, nq in [(2, 11363), (2, 2272)]:
    q = torch.randn(b, nq, 256, device=dev); qp = torch.randn(b, nq, 256, device=dev); mc = torch.randn(b, nq, device=dev)
    with torch.no_grad():
        res = {}
        for fused in (False, True):
            st.FUSED_PRE_ATTENTION = fused
            res[fused] = graph_time(lambda: layer._pre_attention_fast(q, qp, mc), inner=10)
        top = pkg.cabi.topk_desc(mc, 300)
        w_in_t, w_out_t = layer._mha_transposed()
        t, qkv = pkg.cabi.mha_in_proj(q, qp, top, w_in_t, layer.pre_attention.in_proj_bias)
        o = pkg.cabi.attention_qkv(qkv, 8)
        parts = {
            "topk_desc": graph_time(lambda: pkg.cabi.topk_desc(mc, 300)),
            "mha_in_proj": graph_time(lambda: pkg.cabi.mha_in_proj(q, qp, top, w_in_t, layer.pre_attention.in_proj_bias)),
            "attention_qkv": graph_time(lambda: pkg.cabi.attention_qkv(qkv, 8)),
            "out_proj_ln_scatter": graph_time(lambda: pkg.cabi.mha_out_proj_ln_scatter_(q, o, t, w_out_t, layer.pre_attention.out_proj.bias,
                                                                                       layer.pre_norm.weight, layer.pre_norm.bias, 1e-5, top)),
        }
    print(f"pre-attention b={b} nq={nq}: library path {res[False]:.1f} us, fused path {res[True]:.1f} us; parts:",
          {k: round(v, 1) for k, v in parts.items()})
