"""Per-shape timing of the dense projections: hand-written wgmma 3xTF32 GEMM vs cuBLAS 3xTF32 (split pass + TF32
GEMM) vs cuBLAS fp32 SGEMM, on the GEMM shapes of the bench workload (layer 0 and layer 5 query counts)."""
import os, sys, statistics
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import salience_detr_b200 as pkg
dev = "cuda:0"
shapes = [  # (name, M, K, N, relu)
    ("enc_output", 44646, 256, 256, 0), ("value_proj x6", 44646, 256, 1536, 0), ("mask_pred l0", 33600, 256, 256, 0),
    ("proj L0", 22726, 256, 384, 0), ("out_proj L0", 22726, 256, 256, 0), ("class L0", 22726, 256, 91, 0),
    ("ffn1 L0", 22726, 256, 2048, 0), ("ffn2 L0", 22726, 2048, 256, 1),
    ("proj L5", 4544, 256, 384, 0), ("ffn1 L5", 4544, 256, 2048, 0), ("ffn2 L5", 4544, 2048, 256, 1), ("mha 300", 600, 256, 512, 0),
]
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
def timeit(fn, reps=10):
    for _ in range(2): fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b) * 1000)
    return statistics.median(ts)
print(f"{'gemm':14s} {'M':>6s} {'K':>5s} {'N':>5s} | tcgen05 us (K>=1024: SS presplit) | tcgen05 us (persistent raw for all) | cublas3x us | fp32 us | best tcgen05 TF32-TF/s")
tot = {"tcgen05": 0, "3xtf32": 0, "fp32": 0}
for name, M, K, N, relu in shapes:
    x = torch.randn(M, K, device=dev); w = torch.randn(N, K, device=dev) / K ** 0.5; b = torch.randn(N, device=dev)
    r = {}
    for mode in ("tcgen05", "tcgen05-P", "tcgen05-PRE", "3xtf32", "fp32"):
        pkg.gemm.MODE = mode.split("-")[0]
        pkg.gemm.LONG_K_PRESPLIT = mode == "tcgen05"
        pkg.gemm.PRESPLIT_PERSISTENT = mode == "tcgen05-PRE"
        r[mode] = timeit(lambda: pkg.gemm.linear(x, w, b, relu_input=bool(relu)))
        tot[mode] = tot.get(mode, 0) + r[mode]
    print(f"{name:14s} {M:6d} {K:5d} {N:5d} | {r['tcgen05']:9.1f} | {r['tcgen05-P']:9.1f} | pre {r['tcgen05-PRE']:7.1f} | {r['3xtf32']:10.1f} | {r['fp32']:7.1f} | {6*M*N*K/min(r['tcgen05'], r['tcgen05-P'])/1e6:7.1f}")
print("sum", {k: round(v, 1) for k, v in tot.items()})
