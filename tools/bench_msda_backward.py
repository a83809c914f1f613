"""MSDA core forward / backward (the `_C` operator boundary) at the config-2 layer shapes: time per launch and the
fraction of the HBM roofline on algorithmic bytes, and the deterministic (fixed-point) backward next to the atomic one
("det us", "det/bwd").  Results summarised under profiles/."""
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402

dev = torch.device("cuda:0")
try:
    peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    peak = 7700.0
shapes = [(100, 168), (50, 84), (25, 42), (13, 21)]
st = torch.tensor(shapes, dtype=torch.int64, device=dev)
lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
nv = int(st.prod(1).sum())
b, m, d, L, P = 2, 8, 32, 4, 4
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
g = torch.Generator(device="cpu").manual_seed(0)
print("MSDA core at config 2 (b=2, Nv=%d, M=8, D=32, L=4, P=4); HBM peak %.0f GB/s" % (nv, peak))
print("%8s | %10s %10s %8s | %10s %10s %8s | %10s %8s" % ("Nq", "fwd us", "fwd GB/s", "frac", "bwd us", "bwd GB/s", "frac",
                                                         "det us", "det/bwd"))
for nq in (11363, 9090, 6817, 4545, 2272):
    value = torch.randn(b, nv, m, d, generator=g).to(dev)
    # sampling locations as the encoder produces them: reference point + small learned offsets
    ref = torch.rand(b, nq, 1, 1, 1, 2, generator=g)
    loc = (ref + torch.randn(b, nq, m, L, P, 2, generator=g) * 0.03).to(dev)
    attn = torch.randn(b, nq, m, L * P, generator=g).softmax(-1).view(b, nq, m, L, P).to(dev)
    gout = torch.randn(b, nq, m * d, generator=g).to(dev)
    tf, tb, td = [], [], []
    for _ in range(12):
        flush.zero_()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        pkg.cabi.msda_forward(value, st, lsi, loc, attn)
        e[1].record()
        pkg.cabi.msda_backward(value, st, lsi, loc, attn, gout)
        e[2].record()
        torch.cuda.synchronize()
        tf.append(e[0].elapsed_time(e[1]) * 1e3)
        tb.append(e[1].elapsed_time(e[2]) * 1e3)
        flush.zero_()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        pkg.cabi.msda_backward_deterministic(value, st, lsi, loc, attn, gout)  # workspace allocation included (cached)
        e[1].record()
        torch.cuda.synchronize()
        td.append(e[0].elapsed_time(e[1]) * 1e3)
    tf, tb, td = statistics.median(tf[2:]), statistics.median(tb[2:]), statistics.median(td[2:])
    c = m * d
    fwd_bytes = b * (4 * nv * c + nq * (12 * m * L * P + 4 * c))                      # SURVEY 8(d) C_msda
    bwd_bytes = b * (4 * nv * c + nq * (12 * m * L * P + 4 * c)                       # value, loc, attn, grad_out in
                     + 4 * nv * c + nq * 12 * m * L * P)                              # grad_value, grad_loc, grad_attn out
    print("%8d | %10.1f %10.1f %8.3f | %10.1f %10.1f %8.3f | %10.1f %8.2f" % (
        nq, tf, fwd_bytes / tf / 1e3, fwd_bytes / tf / 1e3 / peak, tb, bwd_bytes / tb / 1e3, bwd_bytes / tb / 1e3 / peak,
        td, td / tb))
