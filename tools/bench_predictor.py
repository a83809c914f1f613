"""Salience-filter front (enc_output + LayerNorm + per-level MaskPredictors, without the selection) captured as a CUDA graph:
fused small-level predictor on / off, replayed warm and after an L2 flush."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import salience_detr_b200 as pkg
import salience_detr_b200.salience_transformer as st
from salience_detr_b200.synthetic import build_model, make_inputs

dev = torch.device("cuda:0")
model = build_model().to(dev)
feats, masks, pos = make_inputs("resnet50_800_1333_bs2", seed=0, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
rows_arg = [int(a) for a in sys.argv[1:]] or [4096]
with torch.no_grad():
    plan = model.make_plan(masks)
    b = feats[0].shape[0]
    nv = sum(h * w for h, w in plan.shapes_list)
    x = torch.randn(b, nv, 256, device=dev)

    def scores():
        mem = pkg.gemm.linear(x, model.enc_output.weight, model.enc_output.bias)
        mem = pkg.cabi.add_layernorm(mem, None, model.enc_output_norm.weight, model.enc_output_norm.bias, model.enc_output_norm.eps, out=mem)
        raw = torch.empty(b, nv, device=dev)
        L = len(plan.shapes_list)
        mp = model.enc_mask_predictor
        for lvl in range(L - 1, -1, -1):
            h, w = plan.shapes_list[lvl]
            s0 = plan.level_start[lvl]
            if b * h * w <= st.PREDICTOR_SMALL_ROWS:
                hc, wc = plan.shapes_list[lvl + 1] if lvl != L - 1 else (0, 0)
                coarse = raw[:, plan.level_start[lvl + 1]:plan.level_start[lvl + 1] + hc * wc] if lvl != L - 1 else None
                ln = mp.layer1[0]
                pkg.cabi.mask_predictor_level(mem, s0, h, w, coarse, hc, wc, model.alpha, lvl, ln.weight, ln.bias, ln.eps, *mp.transposed_weights(), raw, s0)
                continue
            m_l = mem[:, s0:s0 + h * w]
            if lvl != L - 1:
                hc, wc = plan.shapes_list[lvl + 1]
                s1 = plan.level_start[lvl + 1]
                m_l = pkg.cabi.score_modulate(mem, s0, h, w, raw[:, s1:s1 + hc * wc], hc, wc, model.alpha, lvl)
            raw[:, s0:s0 + h * w] = mp.forward_fast(m_l).squeeze(-1)
        return raw

    def timed(graph, cold):
        ts = []
        for _ in range(12):
            if cold:
                flush.zero_()
            torch.cuda._sleep(200000)
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); graph.replay(); e.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(e) * 1e3)
        return sorted(ts[2:])[len(ts[2:]) // 2]

    outs = {}
    for rows in [0] + rows_arg:
        st.PREDICTOR_SMALL_ROWS = rows
        for _ in range(2):
            scores()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        n0 = pkg.cabi.launch_count()
        with torch.cuda.graph(g):
            out = scores()
        g.replay(); torch.cuda.synchronize()
        outs[rows] = out.clone()
        print(f"fused predictor for levels of <= {rows} rows: warm {timed(g, False):7.1f} us   L2-flushed {timed(g, True):7.1f} us   max |diff| vs library path {(outs[rows] - outs[0]).abs().max().item():.2e}")
