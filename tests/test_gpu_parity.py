"""GPU parity tests: the sm_90a kernels (called through the C-ABI via salience_detr_b200.cabi) against the
CPU oracle on identical seeded inputs, against the golden fixtures made from the reference, and -- at
BASELINE.json's full sizes -- through size-independent properties.

Tolerances (north_star): top-k / sort indices bit-exact; sampled features <= 1e-3 abs in fp32 (observed ~1e-6,
asserted at 1e-4 or tighter)."""
import os

import numpy as np
import pytest
import torch

from conftest import TINY_CFG, load_golden
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _restore_global_state(pkg):
    """Every test starts from (and leaves) the shipped defaults: gemm.MODE "auto", library options at their defaults --
    so each parity test exercises the configuration a user gets, not whatever an earlier test left behind."""
    mode = pkg.gemm.MODE
    yield
    pkg.gemm.MODE = mode
    pkg.gemm.OWN_KERNEL = os.environ.get("SDETR_GEMM_KERNEL", "f16x3")
    pkg.cabi.lib().sdetr_set_persistent_ctas(0)
    pkg.cabi.set_option("msda_smem_broadcast", 1)


def _msda_inputs(b, shapes, m, d, nq, p, seed):
    g = torch.Generator().manual_seed(seed)
    st = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
    nv = int(st.prod(1).sum())
    L = len(shapes)
    value = torch.randn(b, nv, m, d, generator=g)
    loc = torch.rand(b, nq, m, L, p, 2, generator=g) * 1.2 - 0.1  # exercises out-of-range samples
    attn = torch.randn(b, nq, m, L * p, generator=g).softmax(-1).view(b, nq, m, L, p)
    return value, st, lsi, loc, attn


CASES = [
    # (b, shapes, M, D, Nq, P)         kernel family
    (2, [(16, 20), (8, 10), (4, 5), (2, 3)], 8, 32, 77, 4),          # specialised <32,4,4>
    (1, [(20, 24), (10, 12), (5, 6), (3, 3), (2, 2)], 4, 32, 130, 4),  # specialised <32,5,4> (5-scale)
    (2, [(9, 7), (5, 4), (3, 2), (1, 1)], 2, 64, 33, 4),             # specialised <64,4,4>
    (1, [(7, 5), (4, 3)], 2, 16, 23, 2),                             # generic
    (2, [(6, 6), (3, 3), (2, 2)], 3, 8, 1, 3),                       # generic, single query, odd heads
    (1, [(1, 1), (1, 1), (1, 1), (1, 1)], 8, 32, 5, 4),              # degenerate 1x1 maps
]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("schedule", [0, 1])
def test_msda_forward_vs_oracle(pkg, case, schedule):
    b, shapes, m, d, nq, p = case
    value, st, lsi, loc, attn = _msda_inputs(b, shapes, m, d, nq, p, seed=nq)
    want = orc.c_msda_forward(value, st, lsi, loc, attn)
    args = [t.to(DEV) for t in (value, st, lsi, loc, attn)]
    got = pkg.cabi.msda_forward(*args, schedule=schedule)
    assert got.shape == (b, nq, m * d)
    assert (got.cpu() - want).abs().max() < 1e-4
    # a processing order must not change where results land
    order = torch.stack([torch.randperm(nq, generator=torch.Generator().manual_seed(i)) for i in range(b)]).int()
    got2 = pkg.cabi.msda_forward(*args, query_order=order.to(DEV), schedule=schedule)
    assert torch.equal(got2, got)
    if schedule == 0:
        assert torch.equal(pkg.cabi.msda_forward_plain(*args), got)


@pytest.mark.parametrize("name", ["msda_core_a", "msda_core_b"])
def test_msda_forward_backward_vs_reference_golden(pkg, name):
    g, _ = load_golden(name)
    dv = {k: v.to(DEV) for k, v in g.items()}
    out = pkg.ms_deform_attn_forward(dv["value"], dv["shapes"], dv["lsi"], dv["loc"], dv["attn"], 64)
    assert (out.cpu() - g["out"]).abs().max() < 1e-5
    gv, gl, ga = pkg.ms_deform_attn_backward(dv["value"], dv["shapes"], dv["lsi"], dv["loc"], dv["attn"],
                                             dv["grad_out"], 64)
    assert (gv.cpu() - g["grad_value"]).abs().max() < 1e-4
    assert (ga.cpu() - g["grad_attn"]).abs().max() < 1e-4
    assert (gl.cpu() - g["grad_loc"]).abs().max() / g["grad_loc"].abs().max() < 1e-5


@pytest.mark.parametrize("case", CASES[:4])
def test_msda_backward_vs_oracle(pkg, case):
    b, shapes, m, d, nq, p = case
    value, st, lsi, loc, attn = _msda_inputs(b, shapes, m, d, nq, p, seed=100 + nq)
    gout = torch.randn(b, nq, m * d, generator=torch.Generator().manual_seed(7))
    wv, wl, wa = orc.c_msda_backward(value, st, lsi, loc, attn, gout)
    gv, gl, ga = pkg.cabi.msda_backward(*[t.to(DEV) for t in (value, st, lsi, loc, attn, gout)])
    assert (gv.cpu() - wv).abs().max() < 2e-4 * max(1.0, wv.abs().max().item())
    assert (ga.cpu() - wa).abs().max() < 1e-4
    assert (gl.cpu() - wl).abs().max() / wl.abs().max() < 1e-5


def test_msda_smem_broadcast_variant(pkg):
    """The shared-memory-broadcast build of the specialised kernel gives the same bits as the shuffle build."""
    b, shapes, m, d, nq, p = CASES[0]
    value, st, lsi, loc, attn = _msda_inputs(b, shapes, m, d, nq, p, seed=9)
    args = [t.to(DEV) for t in (value, st, lsi, loc, attn)]
    try:
        outs = []
        for bc in (0, 1):
            pkg.cabi.set_option("msda_smem_broadcast", bc)
            outs.append([pkg.cabi.msda_forward(*args, schedule=s) for s in (0, 1)])
    finally:
        pkg.cabi.set_option("msda_smem_broadcast", 1)  # the library default
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert (outs[1][0].cpu() - orc.c_msda_forward(value, st, lsi, loc, attn)).abs().max() < 1e-4


def test_msda_kernel_variants_agree(pkg):
    """The measured-and-rejected variants stay correct: warp-per-item (option msda_warp_per_item) and TMA-staged
    shared-memory windows (option msda_tma; csrc/msda_forward_tma.cu, incl. its out-of-window global fallback) reproduce
    the default kernel on a tile-ordered head-major launch, fused and plain, 2-d points and 4-d boxes."""
    shapes = [(40, 56), (20, 28), (10, 14), (5, 7)]
    value, st, lsi, loc, attn = [t.to(DEV) for t in _msda_inputs(2, shapes, 8, 32, 777, 4, seed=9)]
    b, nv = value.shape[:2]
    g = torch.Generator().manual_seed(10)
    order = torch.stack([torch.randperm(777, generator=g) for _ in range(b)]).to(torch.int32).to(DEV)
    proj = torch.randn(b, 777, 384, generator=g).to(DEV)
    proj[..., :256] *= 6.0  # offsets of several pixels: some samples leave the staged windows
    ref2 = torch.rand(b, 777, 4, 2, generator=g).to(DEV)
    ref4 = torch.cat([ref2, torch.rand(b, 777, 4, 2, generator=g).to(DEV) * 0.3], -1).contiguous()
    pkg.cabi.msda_set_host_shapes(shapes)

    def run():
        outs = [pkg.cabi.msda_forward(value, st, lsi, loc, attn, query_order=order, schedule=1)]
        for ref in (ref2, ref4):
            outs.append(pkg.cabi.msda_fused_forward(value, nv * 256, 256, 0, st, lsi, ref, proj, 8, 32, 4, 4, nv, order, 1))
        return outs

    try:
        want = run()
        assert (want[0].cpu() - orc.c_msda_forward(value.cpu(), st.cpu(), lsi.cpu(), loc.cpu(), attn.cpu())).abs().max() < 1e-4
        for opt, val in (("msda_warp_per_item", 1), ("msda_warp_per_item", 2), ("msda_tma", 1)):
            pkg.cabi.set_option(opt, val)
            got = run()
            pkg.cabi.set_option(opt, 0)
            for a, w in zip(got, want):
                assert (a - w).abs().max() < 1e-5, (opt, val)
    finally:
        pkg.cabi.set_option("msda_warp_per_item", 0)
        pkg.cabi.set_option("msda_tma", 0)


def test_msda_non_finite_locations_contribute_zero(pkg):
    """A NaN / Inf sampling location is skipped (contributes exactly 0) in the forward as in the reference kernel's branch
    (ms_deform_im2col_cuda.cuh:277) and in the backward -- not 0 * NaN."""
    value, st, lsi, loc, attn = [t.to(DEV) for t in _msda_inputs(2, [(16, 20), (8, 10), (4, 5), (2, 3)], 8, 32, 50, 4, seed=3)]
    bad = loc.clone()
    bad[0, 3, 2, 1, 0, 0] = float("nan")
    bad[1, 7, 5, 3, 2, 1] = float("inf")
    bad[1, 9, 0, 0, 1, :] = -float("inf")
    want = orc.c_msda_forward(value.cpu(), st.cpu(), lsi.cpu(), torch.nan_to_num(bad.cpu(), nan=-9.0, posinf=9.0, neginf=-9.0), attn.cpu())
    for sched in (0, 1):
        out = pkg.cabi.msda_forward(value, st, lsi, bad, attn, schedule=sched)
        assert torch.isfinite(out).all() and (out.cpu() - want).abs().max() < 1e-4


def test_msda_autograd_function(pkg):
    value, st, lsi, loc, attn = _msda_inputs(1, [(6, 5), (3, 3)], 2, 32, 9, 2, seed=3)
    v, l, a = (t.to(DEV).requires_grad_(True) for t in (value, loc, attn))
    out = pkg.MultiScaleDeformableAttnFunction.apply(v, st.to(DEV), lsi.to(DEV), l, a, 64)
    out.sum().backward()
    wv, wl, wa = orc.c_msda_backward(value, st, lsi, loc, attn, torch.ones(1, 9, 64))
    assert (v.grad.cpu() - wv).abs().max() < 1e-4 and (a.grad.cpu() - wa).abs().max() < 1e-4
    assert (l.grad.cpu() - wl).abs().max() / wl.abs().max() < 1e-5


@pytest.mark.parametrize("case", CASES[:4])
@pytest.mark.parametrize("schedule", [0, 1])
def test_msda_fused_forward(pkg, case, schedule):
    """softmax + sampling-location arithmetic fused in (ms_deform_attn.py:322-344)."""
    b, shapes, m, d, nq, p = case
    L = len(shapes)
    g = torch.Generator().manual_seed(5)
    value, st, lsi, _, _ = _msda_inputs(b, shapes, m, d, nq, p, seed=11)
    n = m * L * p
    proj = torch.randn(b, nq, 3 * n, generator=g) * 2
    ref = torch.rand(b, nq, L, 2, generator=g)
    off = proj[..., :2 * n].view(b, nq, m, L, p, 2)
    attn = proj[..., 2 * n:].view(b, nq, m, L * p).softmax(-1).view(b, nq, m, L, p)
    norm = torch.stack([st[:, 1], st[:, 0]], -1).float()
    loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    want = orc.c_msda_forward(value, st, lsi, loc.contiguous(), attn.contiguous())
    vdev = value.to(DEV)
    out, loc_o, attn_o = pkg.cabi.msda_fused_forward(vdev, value[0].numel(), m * d, 0, st.to(DEV), lsi.to(DEV),
                                                      ref.to(DEV), proj.to(DEV), m, d, L, p, value.shape[1],
                                                      schedule=schedule, want_loc_attn=True)
    assert (out.cpu() - want).abs().max() < 1e-4
    assert (loc_o.cpu() - loc).abs().max() < 1e-5
    assert (attn_o.cpu() - attn).abs().max() < 1e-6


# ---- salience filter ------------------------------------------------------------------------------------------
def _select_case(b, shapes, ratios, seed, pad=None, quantize=False):
    g = torch.Generator().manual_seed(seed)
    sizes = [h * w for h, w in shapes]
    starts = [sum(sizes[:i]) for i in range(len(sizes))]
    nv = sum(sizes)
    raw = torch.randn(b, nv, generator=g)
    if quantize:  # many exact ties
        raw = (raw * 4).round() / 4
    mask = torch.zeros(b, nv, dtype=torch.bool)
    if pad:
        for i, frac in enumerate(pad):
            for (h, w), s in zip(shapes, starts):
                m = torch.zeros(h, w, dtype=torch.bool)
                m[:, int(w * (1 - frac)):] = True
                mask[i, s:s + h * w] = m.flatten()
    valid = torch.stack([(~mask[:, s:s + n]).sum(1) for s, n in zip(starts, sizes)], -1)
    k = (valid * torch.tensor(ratios)).int().max(0)[0].tolist()
    return raw, mask, starts, sizes, k


@pytest.mark.parametrize("cfg", [
    dict(b=2, shapes=[(12, 16), (6, 8), (3, 4), (2, 2)], ratios=(0.4, 0.8, 1.0, 1.0), seed=0),
    dict(b=2, shapes=[(12, 16), (6, 8), (3, 4), (2, 2)], ratios=(0.4, 0.8, 1.0, 1.0), seed=1, pad=[0.0, 0.3]),
    dict(b=3, shapes=[(40, 50), (20, 25), (10, 13)], ratios=(0.3, 0.6, 1.0), seed=2, pad=[0.0, 0.1, 0.5], quantize=True),
    dict(b=1, shapes=[(100, 168), (50, 84), (25, 42), (13, 21)], ratios=(0.4, 0.8, 1.0, 1.0), seed=3, pad=[0.008]),
    # k_0 = 10 080 (5 slices of 2048) and K = 40 320 (21 slices): both fit the rank-merge path; the bitonic and radix
    # paths are covered in test_select_paths.py
    dict(b=2, shapes=[(100, 168)], ratios=(0.6,), seed=4, pad=[0.0, 0.2]),
    dict(b=2, shapes=[(200, 336), (100, 168)], ratios=(0.4, 0.8), seed=5, pad=[0.0, 0.1]),
])
def test_salience_select_bit_exact(pkg, cfg):
    raw, mask, starts, sizes, k = _select_case(**cfg)
    widths = [w for _, w in cfg["shapes"]]
    strides = [8 * 2 ** i for i in range(len(widths))]
    wi, ws, wf = orc.c_salience_select(raw, mask, torch.tensor(starts), torch.tensor(sizes), k)
    inds, score, fg, order = pkg.cabi.salience_select(raw.to(DEV), mask.to(torch.uint8).to(DEV), starts, sizes, k,
                                                      widths, strides, 64)
    assert torch.equal(inds.cpu(), wi)              # bit-exact indices incl. the canonical tie order
    assert torch.equal(score.cpu(), ws)
    assert torch.equal(fg.cpu(), wf)
    K = sum(k)
    assert torch.equal(order.long().cpu().sort(1)[0], torch.arange(K).expand(raw.shape[0], K))  # a permutation
    # against torch on the same scores: equal wherever the score is unique (tie order is unspecified in torch)
    for l, (s, n) in enumerate(zip(starts, sizes)):
        filled = raw[:, s:s + n].masked_fill(mask[:, s:s + n], raw[:, s:s + n].min())
        tv, _ = filled.topk(k[l], dim=1)
        mine = score.cpu()  # global order; compare as multisets per level via sorting
        lvl_sel = [(inds[i].cpu() >= s) & (inds[i].cpu() < s + n) for i in range(raw.shape[0])]
        for i in range(raw.shape[0]):
            assert torch.equal(mine[i][lvl_sel[i]], tv[i])
    # prefixes of the processing order
    nqs = [K, int(K * 0.6), int(K * 0.2)]
    pref = pkg.cabi.order_prefixes(order, nqs)
    oc = order.cpu()
    for nq, p in zip(nqs, pref):
        for i in range(raw.shape[0]):
            assert torch.equal(p[i].cpu(), oc[i][oc[i] < nq])


def test_topk_desc(pkg):
    g = torch.Generator().manual_seed(0)
    for seg, n, k in [(2, 11363, 300), (3, 700, 300), (1, 37, 37), (4, 5000, 1), (2, 22323, 3600), (2, 22323, 4096), (1, 9000, 4097)]:
        s = torch.randn(seg, n, generator=g)
        s[:, ::7] = 0.25  # ties
        want = torch.sort(s, dim=1, descending=True, stable=True)[1][:, :k]
        got = pkg.cabi.topk_desc(s.to(DEV), k)
        assert torch.equal(got.cpu(), want)


# ---- token movement / fused elementwise ---------------------------------------------------------------------------
def _levels(shapes):
    st = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
    return st, lsi, int(st.prod(1).sum())


@pytest.mark.parametrize("C", [256, 64])
def test_gather_scatter_background(pkg, C):
    g = torch.Generator().manual_seed(1)
    shapes = [(10, 14), (5, 7), (3, 4), (2, 2)]
    st, lsi, nv = _levels(shapes)
    b, K, nq = 2, 90, 61
    tokens, pos = torch.randn(b, nv, C, generator=g), torch.randn(b, nv, C, generator=g)
    fg = torch.randn(b, nv, generator=g)
    vr = torch.rand(b, 4, 2, generator=g) * 0.5 + 0.5
    sel = torch.stack([torch.randperm(nv, generator=g)[:K] for _ in range(b)])
    inds = sel[:, :nq]  # a prefix view, row stride K
    wq, wqp, wfq, wrq = orc.c_token_gather(tokens, pos, fg, vr, inds, st, lsi, nq)
    d = lambda t: t.to(DEV)
    sel_d = d(sel)
    q, qp, fq, rq = pkg.cabi.token_gather(d(tokens), d(pos), d(fg), d(vr), sel_d[:, :nq], d(st), d(lsi), nq)
    assert torch.equal(q.cpu(), wq) and torch.equal(qp.cpu(), wqp) and torch.equal(fq.cpu(), wfq)
    assert torch.equal(rq.cpu(), wrq)  # same fp32 operations as the reference -> bit-exact
    q2, qp2, fq2, rq2, qs = pkg.cabi.token_gather(d(tokens), d(pos), d(fg), d(vr), sel_d[:, :nq], d(st), d(lsi), nq, want_sum=True)
    assert torch.equal(q2, q) and torch.equal(qp2, qp) and torch.equal(qs.cpu(), wq + wqp)  # + the `with_pos_embed` sum
    # reference-points table of the reference (:417-432) gathered the reference's way
    table = orc.reference_points(shapes, vr)
    want_rq = table.view(b, nv, -1).gather(1, inds[..., None].expand(-1, -1, 8)).view(b, nq, 4, 2)
    assert (rq.cpu() - want_rq).abs().max() < 1e-6
    # scatter: only the first min(focus, nq) rows
    focus = torch.tensor([200, 17], dtype=torch.int32)
    new = torch.randn(b, nq, C, generator=g)
    want = orc.c_token_scatter(tokens.clone(), new, inds, focus)
    tok_d = d(tokens)
    pkg.cabi.token_scatter_(tok_d, d(new), sel_d[:, :nq], d(focus))
    assert torch.equal(tok_d.cpu(), want)
    # background embedding
    mask = torch.rand(b, nv, generator=g) < 0.2
    row, col = torch.rand(40, C // 2, generator=g), torch.rand(40, C // 2, generator=g)
    want = orc.c_background_embed(want.clone(), mask, inds, row, col, st, lsi)
    pkg.cabi.background_embed_(tok_d, d(mask.to(torch.uint8)), sel_d[:, :nq], d(row), d(col), d(st), d(lsi))
    assert torch.equal(tok_d.cpu(), want)


def test_background_embed_table_bounds(pkg):
    """A feature map wider / taller than the learned embedding tables (max_num_embedding, salience_transformer.py:400-407)
    is an index error in the reference (nn.Embedding); here it is a RuntimeError from the host-side check, and the
    kernel clamps, so nothing outside the tables is ever read."""
    b, c, n_emb = 1, 64, 8
    shapes = [(4, 12), (2, 6)]
    st = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.tensor([0, 48], dtype=torch.int64)
    nv = 60
    tok = torch.zeros(b, nv, c, device=DEV)
    mask = torch.zeros(b, nv, dtype=torch.uint8, device=DEV)
    inds = torch.zeros(b, 1, dtype=torch.int64, device=DEV)
    row = torch.rand(n_emb, c // 2, device=DEV)
    col = torch.rand(n_emb, c // 2, device=DEV)
    with pytest.raises(RuntimeError, match="embedding tables hold 8"):
        pkg.cabi.background_embed_(tok, mask, inds, row, col, st.to(DEV), lsi.to(DEV), shapes_host=shapes)
    with pytest.raises(RuntimeError, match="embedding tables hold 8"):  # shapes fetched from the device when not given
        pkg.cabi.background_embed_(tok, mask, inds, row, col, st.to(DEV), lsi.to(DEV))
    # the module path raises the same way (the reference config raises max_num_embedding to 500 for its stride-4 map)
    from salience_detr_b200.synthetic import build_model, make_inputs
    model = build_model(strides=(4, 8, 16, 32), max_num_embedding=200).to(DEV)
    feats, masks, pos = make_inputs("resnet50_5scale_bs2", seed=1, device=DEV)
    with pytest.raises(RuntimeError, match="embedding tables hold 200"), torch.no_grad():
        model.forward_encoder(feats, masks, pos)
    torch.cuda.synchronize()


def test_gelu_colmean(pkg):
    """MaskPredictor middle (reference :40-45): GELU, then the global half replaced by its per-image token mean."""
    g = torch.Generator().manual_seed(21)
    for b, n, c in [(2, 16800, 256), (1, 273, 256), (3, 50, 64), (2, 1000, 96)]:
        z = torch.randn(b, n, c, generator=g)
        half = c // 2
        want = torch.nn.functional.gelu(z.double())
        want[..., half:] = want[..., half:].mean(dim=1, keepdim=True)
        got = pkg.cabi.gelu_colmean_(z.to(DEV), half)
        assert (got.cpu().double() - want).abs().max() < 2e-6
        again = pkg.cabi.gelu_colmean_(z.to(DEV), half)
        assert torch.equal(again, got)  # fixed-order reduction: bit-reproducible


def test_flatten_tokens(pkg):
    g = torch.Generator().manual_seed(6)
    b, C = 2, 64
    shapes = [(13, 21), (7, 11), (4, 6), (2, 3)]
    feats = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
    pos = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
    emb = torch.randn(4, C, generator=g)
    nv = sum(h * w for h, w in shapes)
    keep = (torch.rand(b, nv, generator=g) > 0.2).float()
    want_f = orc.flatten_levels(feats)
    want_p = orc.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, emb)])
    f, p_, x = pkg.cabi.flatten_tokens([t.to(DEV) for t in feats], [t.to(DEV) for t in pos], emb.to(DEV), keep.to(DEV))
    assert torch.equal(f.cpu(), want_f) and torch.equal(p_.cpu(), want_p)
    assert torch.equal(x.cpu(), (want_f + want_p) * keep[..., None])
    # vectorised register-transpose kernel (levels with a token count % 4 == 0) mixed with the tile kernel (the others), wide C,
    # both position-embedding layouts: identical to the oracle and to the tile kernel alone
    for C, shapes in [(256, [(12, 20), (7, 11), (4, 6), (2, 3)]), (320, [(8, 8), (4, 4)]), (32, [(5, 4), (3, 3), (2, 2)])]:
        feats = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
        pos = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
        emb = torch.randn(len(shapes), C, generator=g)
        nv = sum(h * w for h, w in shapes)
        keep = (torch.rand(b, nv, generator=g) > 0.2).float()
        want_f = orc.flatten_levels(feats)
        want_p = orc.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, emb)])
        pos_tok = orc.flatten_levels(pos)
        outs = []
        for vec in (1, 0):
            pkg.cabi.lib().sdetr_flatten_set_vectorized(vec)
            try:
                o1 = pkg.cabi.flatten_tokens([t.to(DEV) for t in feats], [t.to(DEV) for t in pos], emb.to(DEV), keep.to(DEV))
                o2 = pkg.cabi.flatten_tokens_pos([t.to(DEV) for t in feats], pos_tok.to(DEV), emb.to(DEV), keep.to(DEV))
            finally:
                pkg.cabi.lib().sdetr_flatten_set_vectorized(1)
            for o in (o1, o2):
                assert torch.equal(o[0].cpu(), want_f) and torch.equal(o[1].cpu(), want_p), (C, vec)
                assert torch.equal(o[2].cpu(), (want_f + want_p) * keep[..., None]), (C, vec)


def test_attention_qkv(pkg):
    g = torch.Generator().manual_seed(8)
    for b, n, h in [(2, 300, 8), (1, 37, 2), (3, 450, 4)]:
        qk = torch.randn(b, n, 2, h, 32, generator=g)
        v = torch.randn(b, n, h, 32, generator=g)
        want = torch.nn.functional.scaled_dot_product_attention(qk[:, :, 0].transpose(1, 2), qk[:, :, 1].transpose(1, 2),
                                                                v.transpose(1, 2)).transpose(1, 2).reshape(b, n, h * 32)
        qkv = torch.cat([qk.flatten(2), v.flatten(2)], -1).to(DEV)  # packed (b,n,3C) layout of the fused in-projection
        got = pkg.cabi.attention_qkv(qkv, h)
        assert (got.cpu() - want).abs().max() < 2e-5
    with pytest.raises(RuntimeError, match="do not fit in shared memory"):  # K^T, V and the score tile live in smem
        pkg.cabi.attention_qkv(torch.zeros(1, 700, 3 * 4 * 32, device=DEV), 4)


def test_fused_pre_attention_vs_torch_mha(pkg):
    """The three fused kernels of the 300-token pre-attention (gather + in-projection, attention, out-projection +
    residual + LayerNorm + scatter) against nn.MultiheadAttention / nn.LayerNorm in fp64 (reference :366-379)."""
    g = torch.Generator().manual_seed(12)
    c, heads = 256, 8
    mha = torch.nn.MultiheadAttention(c, heads, batch_first=True)
    ln = torch.nn.LayerNorm(c)
    with torch.no_grad():
        for p_ in list(mha.parameters()) + list(ln.parameters()):
            p_.copy_(torch.randn(p_.shape, generator=g) * (0.06 if p_.dim() > 1 else 0.3) + (1.0 if p_ is ln.weight else 0.0))
    for b, nq, k in [(2, 1000, 300), (1, 77, 77), (3, 400, 37)]:
        q = torch.randn(b, nq, c, generator=g)
        qp = torch.randn(b, nq, c, generator=g)
        top = torch.stack([torch.randperm(nq, generator=g)[:k] for _ in range(b)])
        ix = top.unsqueeze(-1).expand(-1, -1, c)
        t = torch.gather(q, 1, ix).double()
        x = t + torch.gather(qp, 1, ix).double()
        m64, l64 = mha.double(), ln.double()
        with torch.no_grad():
            want = q.double().scatter(1, ix, l64(t + m64(x, x, t)[0]))
        mha.float(), ln.float()
        d = lambda z: z.detach().to(DEV).contiguous()
        t_g, qkv = pkg.cabi.mha_in_proj(d(q), d(qp), d(top), d(mha.in_proj_weight.t()), d(mha.in_proj_bias))
        assert torch.equal(t_g.cpu(), torch.gather(q, 1, ix))
        w64, b64 = mha.in_proj_weight.double(), mha.in_proj_bias.double()
        want_qkv = torch.cat([x @ w64[:2 * c].t() + b64[:2 * c], t @ w64[2 * c:].t() + b64[2 * c:]], -1)
        assert (qkv.cpu().double() - want_qkv).abs().max() < 2e-5
        o = pkg.cabi.attention_qkv(qkv, heads)
        out = d(q).clone()
        pkg.cabi.mha_out_proj_ln_scatter_(out, o, t_g, d(mha.out_proj.weight.t()), d(mha.out_proj.bias), d(ln.weight),
                                          d(ln.bias), ln.eps, d(top))
        assert (out.cpu().double() - want).abs().max() < 5e-5, (b, nq, k)
        # with a `query + pos` side buffer: the rewritten rows (and only those) are refreshed
        out2, qs = d(q).clone(), d(q + qp)
        pkg.cabi.mha_out_proj_ln_scatter_(out2, o, t_g, d(mha.out_proj.weight.t()), d(mha.out_proj.bias), d(ln.weight),
                                          d(ln.bias), ln.eps, d(top), d(qp), qs)
        assert torch.equal(out2, out) and torch.equal(qs, out + d(qp))


def test_rows_gather_add_scatter(pkg):
    g = torch.Generator().manual_seed(4)
    b, n, k, C = 2, 500, 300, 256
    src = torch.randn(b, n, C, generator=g)
    idx = torch.stack([torch.randperm(n, generator=g)[:k] for _ in range(b)])
    pos = torch.randn(b, n, C, generator=g)
    t, x = pkg.cabi.rows_gather_add(src.to(DEV), pos.to(DEV), idx.to(DEV))
    want_t = src.gather(1, idx[..., None].expand(-1, -1, C))
    assert torch.equal(t.cpu(), want_t) and torch.equal(x.cpu(), want_t + pos.gather(1, idx[..., None].expand(-1, -1, C)))
    new = torch.randn(b, k, C, generator=g)
    dst = src.to(DEV)
    pkg.cabi.rows_scatter_(dst, idx.to(DEV), new.to(DEV))
    assert torch.equal(dst.cpu(), src.scatter(1, idx[..., None].expand(-1, -1, C), new))


def test_score_modulate_zero_rows_classmax_layernorm(pkg):
    g = torch.Generator().manual_seed(2)
    b, C = 2, 256
    shapes = [(12, 16), (6, 8)]
    nv = 12 * 16 + 6 * 8
    mem = torch.randn(b, nv, C, generator=g)
    raw = torch.randn(b, nv, generator=g)
    alpha = torch.tensor([0.3, -0.2, 0.1])
    up = torch.nn.functional.interpolate(raw[:, 192:].reshape(b, 1, 6, 8), size=(12, 16), mode="bilinear",
                                         align_corners=True)
    want = mem[:, :192] + mem[:, :192] * up.view(b, 1, 192).transpose(1, 2) * alpha[1]
    raw_d = raw.to(DEV)
    got = pkg.cabi.score_modulate(mem.to(DEV), 0, 12, 16, raw_d[:, 192:], 6, 8, alpha.to(DEV), 1)
    assert (got.cpu() - want).abs().max() < 1e-6
    assert (got.cpu() - orc.c_score_modulate(mem[:, :192].contiguous(), raw[:, 192:].contiguous(), float(alpha[1]),
                                             12, 16, 6, 8)).abs().max() < 1e-6
    # zero masked rows of a column slice of a wide buffer
    wide = torch.randn(b, nv, 3 * C, generator=g)
    mask = torch.rand(b, nv, generator=g) < 0.3
    w_d = wide.to(DEV)
    pkg.cabi.zero_masked_rows_(w_d, 3 * C, 3 * C, mask.to(torch.uint8).to(DEV), b * nv)
    assert torch.equal(w_d.cpu(), wide.masked_fill(mask[..., None], 0.0))
    # class max * fg
    logits, fg = torch.randn(b, 77, 91, generator=g), torch.randn(b, 77, generator=g)
    got = pkg.cabi.class_max_times_fg(logits.to(DEV), fg.to(DEV))
    assert torch.equal(got.cpu(), logits.max(-1)[0] * fg)
    padded = torch.zeros(b * 77, 92)
    padded[:, :91] = logits.view(-1, 91)
    got = pkg.cabi.class_max_times_fg(padded.to(DEV)[:, :91].unflatten(0, (b, 77)), fg.to(DEV))  # padded row pitch
    assert torch.equal(got.cpu(), logits.max(-1)[0] * fg)
    # residual + LayerNorm
    for c in (256, 64, 1024):
        x, r = torch.randn(5, 33, c, generator=g), torch.randn(5, 33, c, generator=g)
        gam, bet = torch.randn(c, generator=g), torch.randn(c, generator=g)
        want = torch.nn.functional.layer_norm(x + r, (c,), gam, bet)
        got = pkg.cabi.add_layernorm(x.to(DEV), r.to(DEV), gam.to(DEV), bet.to(DEV))
        assert (got.cpu() - want).abs().max() < 2e-5
        xd = x.to(DEV)
        pkg.cabi.add_layernorm(xd, None, gam.to(DEV), bet.to(DEV), out=xd)  # in place, no residual
        assert (xd.cpu() - torch.nn.functional.layer_norm(x, (c,), gam, bet)).abs().max() < 2e-5


def test_linear_3xtf32_accuracy(pkg):
    """The split-operand TF32 GEMM vs an fp64 reference: ~1e-5 abs on O(1) outputs (tensor-core accumulation is not
    IEEE round-to-nearest, so it sits a few x above cuBLAS SGEMM's ~3e-6) and ~100x better than single-pass TF32."""
    g = torch.Generator().manual_seed(0)
    for rows, K, N in [(4097, 256, 384), (1000, 2048, 256), (333, 256, 91), (50, 64, 1)]:
        x = torch.randn(rows, K, generator=g).to(DEV)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
        b = torch.randn(N, generator=g).to(DEV)
        ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
        pkg.gemm.MODE = "fp32"
        e32 = (pkg.gemm.linear(x, w, b).double() - ref).abs().max().item()
        pkg.gemm.MODE = "3xtf32"
        y = pkg.gemm.linear(x, w, b)
        e3 = (y.double() - ref).abs().max().item()
        pkg.gemm.MODE = "tf32"
        e1 = (pkg.gemm.linear(x, w, b).double() - ref).abs().max().item()
        pkg.gemm.MODE = "3xtf32"
        assert e3 < 8e-5 and e3 < 16 * e32 + 1e-6, (rows, K, N, e3, e32, e1)
        assert e1 > 10 * e3 or K <= 64  # single-pass TF32 is visibly worse: the split is what buys the accuracy
        # fused ReLU on the input operand
        yr = pkg.gemm.linear(x, w, b, relu_input=True)
        assert (yr.double() - torch.nn.functional.linear(x.relu().double(), w.double(), b.double())).abs().max() < 8e-5
    s3 = pkg.cabi.split_tf32(x)
    assert torch.equal(s3[:, :K], s3[:, K:2 * K]) and (s3[:, :K] + s3[:, 2 * K:] - x).abs().max() < 1e-6
    x = torch.randn(7, 64, generator=g).to(DEV)
    s3 = pkg.cabi.split_tf32(x, chunk=16).view(7, 4, 3, 16)  # per-chunk triples
    assert torch.equal(s3[:, :, 0], s3[:, :, 1]) and (s3[:, :, 0] + s3[:, :, 2] - x.view(7, 4, 16)).abs().max() < 1e-6


def test_gemm_persistent_many_tiles_ragged_n(pkg):
    """Persistent kernel with several tiles per CTA and N not a multiple of the 32-column store box (the class head's
    N = 91): the staging boxes of the TMA-store epilogue alternate per issued store.  Repeated, because a box re-used
    too early is a race, not a deterministic error."""
    g = torch.Generator().manual_seed(5)
    for rows, K, N in [(36264, 256, 91), (54396, 256, 96), (40000, 64, 33), (30000, 128, 161)]:
        x = torch.randn(rows, K, generator=g).to(DEV)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
        b = torch.randn(N, generator=g).to(DEV)
        ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
        first = None
        for _ in range(12):
            y = pkg.cabi.gemm_3xtf32_raw(x, w, b)
            assert (y.double() - ref).abs().max().item() < 1e-4, (rows, K, N)
            first = y.clone() if first is None else first
            assert torch.equal(y, first)


def test_gemm_tcgen05_3xtf32(pkg):
    """Hand-written 3xTF32 wgmma GEMM (TMA + in-kernel TF32 split + register accumulator) against an fp64 reference."""
    g = torch.Generator().manual_seed(1)
    for rows, K, N, relu in [(128, 32, 128, False), (300, 256, 384, False), (4097, 256, 256, False), (1000, 2048, 256, True),
                             (333, 256, 91, False), (50, 64, 1, False), (22726, 256, 1536, False), (513, 128, 64, False)]:
        x = torch.randn(rows, K, generator=g).to(DEV)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
        b = torch.randn(N, generator=g).to(DEV)
        w_hi, w_lo = pkg.cabi.split_tf32_pair(w)
        assert (w_hi + w_lo - w).abs().max() < 1e-6
        y = pkg.cabi.gemm_3xtf32(x, w_hi, w_lo, b, relu)
        torch.cuda.synchronize()
        ref = torch.nn.functional.linear((x.relu() if relu else x).double(), w.double(), b.double())
        err = (y.double() - ref).abs().max().item()
        assert err < 3e-4, (rows, K, N, err)  # tensor-core accumulation truncates: grows with K
        # no bias, strided rows (a column slice of a wider buffer)
        wide = torch.randn(rows, K + 32, generator=g).to(DEV)
        y2 = pkg.cabi.gemm_3xtf32(wide[:, 32:], w_hi, w_lo)
        ref2 = wide[:, 32:].double() @ w.double().t()
        assert (y2.double() - ref2).abs().max() < 1e-4
        # the raw-weight form (W split in the kernel) and the pre-split persistent entry point: same arithmetic
        y4 = pkg.cabi.gemm_3xtf32_raw(x, w, b, int(relu))
        assert y4.shape == y.shape and (y4.double() - ref).abs().max() < 3e-4
        y5 = pkg.cabi.gemm_3xtf32_pre(x, w_hi, w_lo, b, int(relu))  # persistent kernel, pre-split weight: same arithmetic
        assert torch.equal(y5, y4)
    prev = pkg.gemm.MODE
    try:
        pkg.gemm.MODE = "tcgen05"
        x = torch.randn(2, 77, 256, generator=g).to(DEV)
        w = torch.randn(384, 256, generator=g).to(DEV) / 16
        y = pkg.gemm.linear(x, w, None)
        assert y.shape == (2, 77, 384) and (y.double() - x.double() @ w.double().t()).abs().max() < 1e-4
    finally:
        pkg.gemm.MODE = prev


def test_gemm_f16x3_accuracy_and_range(pkg):
    """3xFP16 persistent kernel (wgmma .f16 on hi/lo fp16 pairs, power-of-two range scalings) against an fp64
    reference: the same fp32-class error as 3xTF32 / SGEMM on O(1) data, across the documented activation range
    (2^-7 .. 4094 relative accuracy, absolute floor below), with the fused input activations, ragged N, strided rows,
    many tiles per CTA, and bit-reproducible."""
    g = torch.Generator().manual_seed(7)
    F = torch.nn.functional
    for rows, K, N, act in [(128, 64, 128, None), (300, 256, 384, None), (4097, 256, 256, None), (1000, 2048, 256, "relu"),
                            (333, 256, 91, None), (50, 64, 1, None), (22726, 256, 1536, None), (513, 128, 64, "gelu"),
                            (36264, 256, 91, None), (40000, 64, 33, None)]:
        x = torch.randn(rows, K, generator=g).to(DEV)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
        b = torch.randn(N, generator=g).to(DEV)
        w_hi, w_lo, sc = pkg.cabi.split_f16_pair(w)
        assert 2 ** 13 <= float(w.abs().max()) * sc < 2 ** 14
        assert ((w_hi.float() + w_lo.float()) / sc - w).abs().max() < 2e-7 * float(w.abs().max())  # 22-bit weight
        y = pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc, b, {None: 0, "relu": 1, "gelu": 2}[act])
        xa = x.double() if act is None else (F.relu(x.double()) if act == "relu" else F.gelu(x.double()))
        ref = F.linear(xa, w.double(), b.double())
        err = (y.double() - ref).abs().max().item()
        pkg.gemm.MODE = "fp32"
        e32 = (pkg.gemm.linear(x if act is None else (F.relu(x) if act == "relu" else F.gelu(x)), w, b).double() - ref).abs().max().item()
        assert err < 3e-4 and err < 32 * e32 + 1e-6, (rows, K, N, err, e32)
        assert torch.equal(pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc, b, {None: 0, "relu": 1, "gelu": 2}[act]), y)
    # the benched shapes and the awkward ones: wide N, long K, one-panel problems, ragged N, many tiles per CTA (also with
    # the persistent grid capped at a few CTAs); bit-reproducible whatever the grid
    for rows, K, N, act in [(22726, 256, 2048, 0), (4544, 256, 2048, 1), (44646, 256, 1536, 0), (20000, 128, 640, 2),
                            (19000, 64, 384, 0), (18180, 256, 384, 0), (40000, 192, 300, 0), (22726, 2048, 256, 1), (129, 64, 128, 0),
                            (385, 256, 91, 0), (100, 128, 256, 0), (36264, 256, 91, 2), (4544, 256, 384, 0)]:
        x = torch.randn(rows, K, generator=g).to(DEV)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV)
        b = torch.randn(N, generator=g).to(DEV)
        w_hi, w_lo, sc = pkg.cabi.split_f16_pair(w)
        y0 = pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc, b, act)
        xa = x.double() if act == 0 else (F.relu(x.double()) if act == 1 else F.gelu(x.double()))
        assert (y0.double() - F.linear(xa, w.double(), b.double())).abs().max() < 1e-4, (rows, K, N)
        pkg.cabi.lib().sdetr_set_persistent_ctas(7)
        y1 = pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc, b, act)
        pkg.cabi.lib().sdetr_set_persistent_ctas(0)
        assert torch.equal(y0, y1), (rows, K, N)
        for _ in range(3):
            assert torch.equal(pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc, b, act), y0)
    # range: tiny, huge and mixed-magnitude activations; relative error of the result stays fp32-class
    K, N = 256, 256
    w = (torch.randn(N, K, generator=g) / 16).to(DEV)
    w_hi, w_lo, sc = pkg.cabi.split_f16_pair(w)
    for scale in (1e-3, 1e-2, 1.0, 100.0, 3000.0):
        x = (torch.randn(2000, K, generator=g) * scale).clamp(-4000, 4000).to(DEV)
        y = pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc)
        ref = x.double() @ w.double().t()
        rel = ((y.double() - ref).abs().max() / ref.abs().max()).item()
        assert rel < (2e-6 if scale >= 1e-2 else 2e-5), (scale, rel)  # below 2^-7 the absolute floor 2^-29 takes over
    x = torch.randn(2000, K, generator=g).to(DEV) * torch.logspace(-4, 2, K).to(DEV)  # 6 decades inside one row (|x| < 4094)
    y = pkg.cabi.gemm_f16x3_pre(x, w_hi, w_lo, sc)
    ref = x.double() @ w.double().t()
    assert ((y.double() - ref).abs().max() / ref.abs().max()).item() < 2e-6
    # strided rows (a column slice of a wider buffer), no bias; weight with a large dynamic range
    wide = torch.randn(777, K + 64, generator=g).to(DEV)
    w2 = (torch.randn(N, K, generator=g) * torch.logspace(-6, 0, K)).to(DEV)
    h2, l2, s2 = pkg.cabi.split_f16_pair(w2)
    y2 = pkg.cabi.gemm_f16x3_pre(wide[:, 64:], h2, l2, s2)
    ref2 = wide[:, 64:].double() @ w2.double().t()
    assert ((y2.double() - ref2).abs().max() / ref2.abs().max()).item() < 2e-6
    # gemm.linear routes to it in the default mode, and to 3xTF32 when K % 64 != 0
    pkg.gemm.MODE, pkg.gemm.OWN_KERNEL = "auto", "f16x3"
    x = torch.randn(2, 3000, 256, generator=g).to(DEV)
    y = pkg.gemm.linear(x, w, None)
    assert y.shape == (2, 3000, 256) and (y.double() - x.double() @ w.double().t()).abs().max() < 1e-4
    w96 = torch.randn(128, 96, generator=g).to(DEV) / 10
    x96 = torch.randn(5000, 96, generator=g).to(DEV)
    assert (pkg.gemm.linear(x96, w96).double() - x96.double() @ w96.double().t()).abs().max() < 1e-4


# ---- module level ---------------------------------------------------------------------------------------------------
@pytest.fixture(params=["fp32", "3xtf32", "tcgen05", "auto"])
def gemm_mode(pkg, request):
    prev = pkg.gemm.MODE
    pkg.gemm.MODE = request.param
    yield request.param
    pkg.gemm.MODE = prev


def _tiny_model(pkg, sd):
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(64, 128, 0.0, 2, topk_sa=20), 3, 40)
    tr = pkg.SalienceTransformer(enc, num_classes=11, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
                                 layer_filter_ratio=(1.0, 0.6, 0.3)).to(DEV).eval()
    missing = tr.load_state_dict(sd, strict=False)
    assert not missing.missing_keys
    return tr


def _golden_inputs(g):
    return ([g[f"feat{i}"].to(DEV) for i in range(4)], [g[f"mask{i}"].to(DEV) for i in range(4)],
            [g[f"pos{i}"].to(DEV) for i in range(4)])


def test_msda_module_vs_reference_golden(pkg, gemm_mode):
    g, sd = load_golden("msda_module")
    tol = 1e-5 if gemm_mode == "fp32" else 1e-4
    mod = pkg.MultiScaleDeformableAttention(64, 4, 2, 4).to(DEV).eval()
    mod.load_state_dict(sd)
    args = [g[k].to(DEV) for k in ("query", "ref", "value", "shapes", "lsi", "mask")]
    with torch.no_grad():
        out = mod(*args)                       # fused inference path
    assert (out.cpu() - g["out"]).abs().max() < tol
    out2 = mod(*args)                          # autograd path (parameters require grad)
    assert (out2.detach().cpu() - g["out"]).abs().max() < 1e-5
    out2.sum().backward()
    assert mod.sampling_offsets.weight.grad is not None and torch.isfinite(mod.value_proj.weight.grad).all()


def test_msda_module_reference_boxes(pkg):
    """4-d reference points (the decoder's reference-box branch, ms_deform_attn.py:345-349) through the module."""
    g = torch.Generator().manual_seed(12)
    mod = pkg.MultiScaleDeformableAttention(64, 4, 2, 4).to(DEV).eval()
    with torch.no_grad():
        mod.sampling_offsets.weight.normal_(0, 0.05, generator=None)
        mod.attention_weights.weight.normal_(0, 0.5)
    shapes = [(9, 12), (5, 6), (3, 3), (2, 2)]
    st, lsi, nv = _levels(shapes)
    b, nq = 2, 21
    query, value = torch.randn(b, nq, 64, generator=g), torch.randn(b, nv, 64, generator=g)
    boxes = torch.rand(b, nq, 4, 4, generator=g) * 0.5 + 0.25
    mask = torch.rand(b, nv, generator=g) < 0.1
    sd = {k: v.detach().cpu() for k, v in mod.state_dict().items()}
    v = torch.nn.functional.linear(value, sd["value_proj.weight"], sd["value_proj.bias"]).masked_fill(mask[..., None], 0).view(b, nv, 2, 32)
    off = torch.nn.functional.linear(query, sd["sampling_offsets.weight"], sd["sampling_offsets.bias"]).view(b, nq, 2, 4, 4, 2)
    att = torch.nn.functional.linear(query, sd["attention_weights.weight"], sd["attention_weights.bias"]).view(b, nq, 2, 16).softmax(-1).view(b, nq, 2, 4, 4)
    loc = boxes[:, :, None, :, None, :2] + off / 4 * boxes[:, :, None, :, None, 2:] * 0.5
    want = torch.nn.functional.linear(orc.c_msda_forward(v.contiguous(), st, lsi, loc.contiguous(), att.contiguous()),
                                      sd["output_proj.weight"], sd["output_proj.bias"])
    with torch.no_grad():
        got = mod(query.to(DEV), boxes.to(DEV), value.to(DEV), st.to(DEV), lsi.to(DEV), mask.to(DEV))
    assert (got.cpu() - want).abs().max() < 1e-4


def test_five_scale_stress_geometry(pkg):
    """salience_detr_resnet50_5scale geometry (strides 4/8/16/32, Nv = 89 250, K = 45 330 with the 800x1333-in-800x1344
    padding mask; 45 570 for an all-valid mask): the selection (25 slices of 2048 and 2464 cell bins, so the rank-merge
    path) stays bit-exact with the oracle and the encoder half runs end to end."""
    from salience_detr_b200.synthetic import build_model, make_inputs
    torch.cuda.synchronize()  # surface any earlier asynchronous error here, not inside this test
    model = build_model(strides=(4, 8, 16, 32)).to(DEV)
    feats, masks, pos = make_inputs("resnet50_5scale_bs2", seed=1, device=DEV)
    assert sum(f.shape[2] * f.shape[3] for f in feats) == 89250
    with torch.no_grad():
        mem, aux = model.forward_encoder(feats, masks, pos)
    plan = aux["plan"]
    assert plan.num_selected == 45330 and mem.shape == (2, 89250, 256) and torch.isfinite(mem).all()
    wi, ws, wf = orc.c_salience_select(aux["raw_score"].cpu(), plan.mask_flat.cpu(), plan.level_start_index.cpu(),
                                       torch.tensor(plan.level_size), plan.level_token_nums)
    assert torch.equal(aux["selected_inds"].cpu(), wi) and torch.equal(aux["foreground_score"].cpu(), wf)
    # same selection re-used in strict fp32-GEMM mode: the layers agree within the 3xTF32 tolerance
    prev = pkg.gemm.MODE
    try:
        pkg.gemm.MODE = "fp32"
        feat = pkg.flatten_levels(feats)
        lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, model.level_embeds)])
        with torch.no_grad():
            mem32 = model.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat,
                                  spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index,
                                  valid_ratios=plan.valid_ratios, foreground_score=aux["foreground_score"],
                                  focus_token_nums=plan.focus_token_nums,
                                  foreground_inds=[aux["selected_inds"][:, :n] for n in plan.layer_num_query],
                                  multi_level_masks=masks)
    finally:
        pkg.gemm.MODE = prev
    assert (mem - mem32).abs().max() < 5e-3


@pytest.mark.parametrize("use_order", [False, True])
def test_encoder_half_vs_reference_golden_even(pkg, use_order, gemm_mode):
    """Tie-free batch: bit-exact selected indices, memory within fp32 round-off of the reference.
    (Index equality at module level needs bit-compatible scores -- SURVEY.md 8(a) "parity levels" -- so it is
    asserted in fp32-GEMM mode; in 3xTF32 mode the scores move by ~1e-5 and near-ties may swap.)"""
    g, sd = load_golden("encoder_tiny_even")
    tr = _tiny_model(pkg, sd)
    feats, masks, pos = _golden_inputs(g)
    with torch.no_grad():
        mem, aux = tr.forward_encoder(feats, masks, pos, use_order=use_order)
    if gemm_mode == "fp32":
        assert torch.equal(aux["selected_inds"].cpu(), g["selected_inds"])
    else:
        same = (aux["selected_inds"].cpu() == g["selected_inds"]).float().mean().item()
        assert same > 0.9, same
    assert aux["plan"].layer_num_query == g["layer_num_query"].tolist()
    assert torch.equal(aux["plan"].focus_token_nums.cpu().long(), g["focus_token_nums"].long())
    assert (aux["foreground_score"].cpu() - g["foreground_score"]).abs().max() < (1e-5 if gemm_mode == "fp32" else 2e-4)
    if gemm_mode == "fp32" or torch.equal(aux["selected_inds"].cpu(), g["selected_inds"]):
        assert (mem.cpu() - g["memory"]).abs().max() < (2e-4 if gemm_mode == "fp32" else 2e-3)
    # plan reuse: second call with the cached plan (no host sync) gives the same bits
    with torch.no_grad():
        mem2, _ = tr.forward_encoder(feats, masks, pos, plan=aux["plan"], use_order=use_order)
    assert torch.equal(mem2, mem)


def test_encoder_half_ragged_and_injected_indices(pkg, gemm_mode):
    """Ragged batch (padded tokens tie): selection equals the oracle's canonical order bit for bit; with the
    reference's own indices injected the encoder reproduces the reference memory."""
    g, sd = load_golden("encoder_tiny_ragged")
    tr = _tiny_model(pkg, sd)
    feats, masks, pos = _golden_inputs(g)
    with torch.no_grad():
        mem, aux = tr.forward_encoder(feats, masks, pos)
    cpu_in = ([g[f"feat{i}"] for i in range(4)], [g[f"mask{i}"] for i in range(4)], [g[f"pos{i}"] for i in range(4)])
    omem, ofilt = orc.encoder_half_forward(sd, *cpu_in, TINY_CFG, core="c", use_c_helpers=True)
    assert (aux["raw_score"].cpu() - ofilt["raw_score"]).abs().max() < (1e-5 if gemm_mode == "fp32" else 2e-4)
    # the oracle's indices on the GPU's own scores (scores differ by round-off between CPU and cuBLAS)
    plan = aux["plan"]
    wi, _, _ = orc.c_salience_select(aux["raw_score"].cpu(), plan.mask_flat.cpu(), plan.level_start_index.cpu(),
                                     torch.tensor(plan.level_size), plan.level_token_nums)
    assert torch.equal(aux["selected_inds"].cpu(), wi)
    # inject the reference's indices into the encoder
    ref_inds = g["selected_inds"].to(DEV)
    feat = pkg.flatten_levels(feats)
    lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, tr.level_embeds)])
    with torch.no_grad():
        mem_inj = tr.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat,
                             spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index,
                             valid_ratios=plan.valid_ratios, foreground_score=g["foreground_score"].to(DEV),
                             focus_token_nums=plan.focus_token_nums,
                             foreground_inds=[ref_inds[:, :n] for n in plan.layer_num_query], multi_level_masks=masks)
    assert (mem_inj.cpu() - g["memory"]).abs().max() < (2e-4 if gemm_mode == "fp32" else 2e-3)


def test_config1_encoder_half_vs_oracle(pkg):
    """BASELINE.json configs[0] (512x512, bs=1, Nv=5440, K=2777) at the real model dimensions (C=256, 8 heads, 6 layers,
    topk_sa=300): filter scores against the CPU oracle, then -- with the oracle's own indices injected, so both sides
    process the same tokens -- the encoder memory within the north-star tolerance (1e-3 abs), in strict fp32 and in the
    default 3xTF32 GEMM mode."""
    from salience_detr_b200.synthetic import build_model, make_inputs
    model = build_model().to(DEV)
    feats, masks, pos = make_inputs("cpu_512", seed=3, device=DEV)
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    cfg = dict(heads=8, points=4, topk_sa=300, num_layers=6, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
               layer_filter_ratio=(1.0, 0.8, 0.6, 0.6, 0.4, 0.2))
    omem, ofilt = orc.encoder_half_forward(sd, [f.cpu() for f in feats], [m.cpu() for m in masks], [p.cpu() for p in pos],
                                           cfg, core="c", use_c_helpers=True)
    assert ofilt["selected_inds"].shape == (1, 2777) and ofilt["layer_num_query"] == [2777, 2221, 1666, 1666, 1110, 555]
    oinds, ofg = ofilt["selected_inds"].to(DEV), ofilt["foreground_score"].to(DEV)
    for mode, tol_score, tol_mem in (("fp32", 2e-5, 1e-3), ("auto", 2e-4, 1e-3)):
        pkg.gemm.MODE = mode
        with torch.no_grad():
            mem, aux = model.forward_encoder(feats, masks, pos)
        plan = aux["plan"]
        assert plan.num_selected == 2777 and plan.layer_num_query == ofilt["layer_num_query"]
        assert (aux["raw_score"].cpu() - ofilt["raw_score"]).abs().max() < tol_score
        got, want = set(aux["selected_inds"][0].tolist()), set(ofilt["selected_inds"][0].tolist())
        assert len(got & want) >= 2777 - 8  # near-ties at the budget boundary may swap (scores differ by round-off)
        feat = pkg.flatten_levels(feats)
        lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, model.level_embeds)])
        with torch.no_grad():
            mem_inj = model.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat,
                                    spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index,
                                    valid_ratios=plan.valid_ratios, foreground_score=ofg,
                                    focus_token_nums=plan.focus_token_nums,
                                    foreground_inds=[oinds[:, :n] for n in plan.layer_num_query], multi_level_masks=masks)
        err = (mem_inj.cpu() - omem).abs().max().item()
        assert err < tol_mem, (mode, err)


def test_encoder_runner_graph_matches_eager(pkg):
    """EncoderRunner (one CUDA graph, value projection on a parallel branch) and HostPipeline (double-buffered host I/O)
    reproduce the eager forward bit for bit."""
    from salience_detr_b200.runner import EncoderRunner, HostPipeline
    g, sd = load_golden("encoder_tiny_ragged")
    tr = _tiny_model(pkg, sd)
    feats, masks, pos = _golden_inputs(g)
    with torch.no_grad():
        want, _ = tr.forward_encoder(feats, masks, pos)
    runner = EncoderRunner(tr, feats, masks, pos)
    assert runner.graph is not None and runner.launches_per_step > 0
    for _ in range(3):
        got = runner.step()
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    runner.bind_host([f.cpu() for f in feats], [p.cpu() for p in pos])
    host = runner.run_host()  # asynchronous on the runner's stream: synchronise before reading the pinned buffer
    runner.stream.synchronize()
    assert torch.equal(host.to(DEV), want)
    pipe = HostPipeline(tr, feats, masks, pos, depth=2)
    outs = {}
    batch = ([f.cpu().pin_memory() for f in feats], [p.cpu().pin_memory() for p in pos])
    n = pipe.run([batch] * 5, on_output=lambda i, h: outs.__setitem__(i, h.clone()))
    assert n == 5 and sorted(outs) == [0, 1, 2, 3, 4]  # every batch is handed out, in order (the last two at the drain)
    for h in list(outs.values()) + pipe.host_out:
        assert torch.equal(h.to(DEV), want)


def test_fresh_mask_pipeline(pkg):
    """FreshMaskPipeline: batches with DIFFERENT padding masks (each pays its own plan and an eager forward; copies, plans and
    forwards of consecutive batches overlap) give exactly the eager result of their own masks, in order."""
    from salience_detr_b200.runner import FreshMaskPipeline
    from salience_detr_b200.position_encoding import PositionEmbeddingSine
    g, sd = load_golden("encoder_tiny_ragged")
    tr = _tiny_model(pkg, sd)
    tr.attach_position_embedding(PositionEmbeddingSine(tr.embed_dim // 2, temperature=10000, normalize=True, offset=-0.5))
    feats, masks, _ = _golden_inputs(g)
    masks_b = [torch.zeros_like(m) for m in masks]                     # no padding at all
    masks_c = [m.clone() for m in masks]
    for m in masks_c:                                                  # a different ragged padding: last column block padded
        m[:, :, -max(1, m.shape[2] // 3):] = True
    feats2 = [f * 0.5 + 0.1 for f in feats]
    variants = [(feats, masks), (feats2, masks_b), (feats, masks_c), (feats2, masks)]
    wants = []
    with torch.no_grad():
        for f, m in variants:
            wants.append(tr.forward_encoder(f, m, None)[0].clone())
    assert not torch.equal(wants[0], wants[2])
    pipe = FreshMaskPipeline(tr, feats, masks, depth=2)
    pin = lambda ts: [t.cpu().pin_memory() for t in ts]  # noqa: E731
    batches = [(pin(f), pin(m)) for f, m in variants] * 2
    outs = {}
    n = pipe.run(batches, on_output=lambda i, h: outs.__setitem__(i, h.clone()))
    assert n == 8 and sorted(outs) == list(range(8))
    for i in range(8):
        assert torch.equal(outs[i].to(DEV), wants[i % 4]), i


def test_encoder_training_path_gradients(pkg):
    """Training path (torch autograd around the MSDA forward / backward kernels) against the REFERENCE's own autograd
    (tests/golden/encoder_tiny_even_grads.npz, oracle/make_golden.py::make_encoder_tiny_grads): loss and the gradient of
    every parameter the loss reaches, and of the input feature maps."""
    g, sd = load_golden("encoder_tiny_even")
    gg, _ = load_golden("encoder_tiny_even_grads")
    tr = _tiny_model(pkg, sd).train()
    feats, masks, pos = _golden_inputs(g)
    feats = [f.clone().requires_grad_(True) for f in feats]
    mem, _ = tr.forward_encoder(feats, masks, pos)
    assert (mem.detach().cpu() - g["memory"]).abs().max() < 2e-4  # dropout = 0 -> same values
    loss = mem.square().mean()
    assert abs(loss.item() - gg["loss"].item()) < 1e-5
    loss.backward()
    params = dict(tr.named_parameters())
    checked = 0
    for key, want in gg.items():
        if key.startswith("grad."):
            got = params[key[5:]].grad
        elif key.startswith("grad_feat"):
            got = feats[int(key[9:])].grad
        else:
            continue
        assert got is not None, key
        err = (got.cpu() - want).abs().max().item()
        assert err <= 2e-3 * want.abs().max().item() + 1e-7, (key, err, want.abs().max().item())
        checked += 1
    assert checked == len(gg) - 1 and checked >= 70
    for name, p in params.items():  # parameters the reference's loss does not reach stay without gradient here too
        if ("grad." + name) not in gg:
            assert p.grad is None or p.grad.abs().max() == 0, name


# ---- error behaviour of the boundary (reference: AT_ASSERTM -> RuntimeError, .cu:20-30,42-44) ---------------------------
def test_boundary_errors(pkg):
    value, st, lsi, loc, attn = [t.to(DEV) for t in _msda_inputs(3, [(4, 4), (2, 2)], 2, 32, 5, 2, seed=0)]
    with pytest.raises(RuntimeError, match="contiguous"):
        pkg.ms_deform_attn_forward(value.transpose(1, 2), st, lsi, loc, attn, 64)
    with pytest.raises(RuntimeError, match="CUDA"):
        pkg.ms_deform_attn_forward(value.cpu(), st, lsi, loc, attn, 64)
    with pytest.raises(RuntimeError, match="im2col_step"):
        pkg.ms_deform_attn_forward(value, st, lsi, loc, attn, 2)  # 3 % 2 != 0
    with pytest.raises(RuntimeError, match="k="):
        pkg.cabi.topk_desc(torch.randn(1, 10, device=DEV), 11)
    with pytest.raises(RuntimeError, match="level"):
        pkg.cabi.salience_select(torch.randn(1, 10, device=DEV), torch.zeros(1, 10, dtype=torch.uint8, device=DEV),
                                 [0, 5], [5, 5], [6, 1])
    # empty query set is a no-op, not an error
    out = pkg.cabi.msda_forward(value, st, lsi, loc[:, :0].contiguous(), attn[:, :0].contiguous())
    assert out.shape == (3, 0, 64)


# ---- full BASELINE sizes: size-independent properties + oracle spot checks -------------------------------------------------
def test_full_size_config2_properties(pkg):
    """salience_detr_resnet50_800_1333, bs=2: levels (100,168),(50,84),(25,42),(13,21), Nv=22323, K=11363."""
    shapes = [(100, 168), (50, 84), (25, 42), (13, 21)]
    st, lsi, nv = _levels(shapes)
    assert nv == 22323
    g = torch.Generator().manual_seed(0)
    b, m, d, nq = 2, 8, 32, 11363
    value = torch.randn(b, nv, m, d, generator=g)
    loc = torch.rand(b, nq, m, 4, 4, 2, generator=g) * 1.1 - 0.05
    attn = torch.randn(b, nq, m, 16, generator=g).softmax(-1).view(b, nq, m, 4, 4)
    dv = [t.to(DEV) for t in (value, st, lsi, loc, attn)]
    out = pkg.cabi.msda_forward(*dv)
    want = orc.c_msda_forward(value, st, lsi, loc, attn)
    assert (out.cpu() - want).abs().max() < 1e-4
    # linearity in value and in the attention weights; idempotence across schedules/orders
    out2 = pkg.cabi.msda_forward(dv[0] * 2, dv[1], dv[2], dv[3], dv[4] * 0.5, schedule=1)
    assert (out2 - out).abs().max() < 1e-5
    # constant value field + weights summing to 1 + in-range samples -> the constant comes back
    loc_in = torch.rand(b, nq, m, 4, 4, 2, generator=g) * 0.8 + 0.1
    ones = torch.ones_like(dv[0])
    o = pkg.cabi.msda_forward(ones, dv[1], dv[2], loc_in.to(DEV), dv[4])
    assert (o - 1).abs().max() < 1e-5
    # selection at full size: sortedness, uniqueness, level budgets
    raw = torch.randn(b, nv, generator=g)
    mask = torch.zeros(b, 100, 168, dtype=torch.bool)
    mask[:, :, 167:] = True
    mask_flat = torch.cat([mask.flatten(1), torch.zeros(b, nv - 16800, dtype=torch.bool)], 1)
    starts, sizes, k = lsi.tolist(), st.prod(1).tolist(), [6680, 3360, 1050, 273]
    inds, score, fg, order = pkg.cabi.salience_select(raw.to(DEV), mask_flat.to(torch.uint8).to(DEV), starts, sizes, k,
                                                      [168, 84, 42, 21], [8, 16, 32, 64], 128)
    sc, ic = score.cpu(), inds.cpu()
    assert (sc[:, 1:] <= sc[:, :-1]).all()
    for i in range(b):
        assert ic[i].unique().numel() == 11363
        assert [int(((ic[i] >= s) & (ic[i] < s + n)).sum()) for s, n in zip(starts, sizes)] == k
    wi, ws, wf = orc.c_salience_select(raw, mask_flat, lsi, st.prod(1), k)
    assert torch.equal(ic, wi) and torch.equal(sc, ws) and torch.equal(fg.cpu(), wf)


def test_encoder_half_c256_vs_reference_golden(pkg):
    """The reference itself at its real width (C = 256, 8 heads of 32, 4080 tokens per image; fixture made by
    oracle/make_golden.py, weights / inputs regenerated from seeds): this geometry takes the paths specialised for the
    real model -- fused pre-attention, persistent tensor-core GEMM, fused GELU + token mean.  Scores and selection
    against the reference; with the reference's indices injected, the encoder memory within 1e-3 (north-star bound)."""
    from conftest import C256_CFG, load_c256_golden
    g, sd, (feats, masks, pos) = load_c256_golden()
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(256, 256, 0.0, 8, topk_sa=64), 2, 80)
    tr = pkg.SalienceTransformer(enc, num_classes=11, level_filter_ratio=C256_CFG["level_filter_ratio"],
                                 layer_filter_ratio=C256_CFG["layer_filter_ratio"]).to(DEV).eval()
    missing = tr.load_state_dict(sd, strict=False).missing_keys  # the two ratio buffers keep their constructor values
    assert sorted(missing) == ["layer_filter_ratio", "level_filter_ratio"]
    feats, masks, pos = [f.to(DEV) for f in feats], [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]
    ref_inds, ref_fg = g["selected_inds"].to(DEV), g["foreground_score"].to(DEV)
    rows_ix = g["memory_rows_index"].to(DEV)
    for mode, tol_score, max_swaps, tol_mem in (("fp32", 2e-5, 8, 1e-3), ("auto", 3e-4, 40, 1e-3)):
        pkg.gemm.MODE = mode  # restored by the autouse fixture
        with torch.no_grad():
            mem, aux = tr.forward_encoder(feats, masks, pos)
        plan = aux["plan"]
        assert plan.layer_num_query == g["layer_num_query"].tolist()
        assert (aux["foreground_score"] - ref_fg).abs().max() < tol_score, mode
        for i in range(2):  # near-ties at the budget boundary may swap (scores differ by round-off), nothing else
            got, want = set(aux["selected_inds"][i].tolist()), set(g["selected_inds"][i].tolist())
            assert len(got & want) >= len(want) - max_swaps, (mode, len(got & want))
        feat = pkg.flatten_levels(feats)
        lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, tr.level_embeds)])
        with torch.no_grad():
            mem_inj = tr.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat,
                                 spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index,
                                 valid_ratios=plan.valid_ratios, foreground_score=ref_fg,
                                 focus_token_nums=plan.focus_token_nums,
                                 foreground_inds=[ref_inds[:, :n] for n in plan.layer_num_query], multi_level_masks=masks)
        rows = torch.gather(mem_inj, 1, rows_ix[..., None].expand(-1, -1, 256))
        assert (rows.cpu() - g["memory_rows"]).abs().max() < tol_mem, mode
        assert (mem_inj.mean(-1).cpu() - g["memory_row_mean"]).abs().max() < tol_mem
        assert (mem_inj.abs().amax(-1).cpu() - g["memory_row_absmax"]).abs().max() < 2 * tol_mem


def test_mask_plan_and_sine_position_tokens(pkg):
    """Device-side plan (sdetr_mask_plan: budgets, valid ratios, keep mask, normalised coordinates) against the torch
    restatement of the reference arithmetic (salience_transformer.py:116-121,161-165; base_transformer.py:48-56,74-110),
    and the fused sine position embedding in token layout against PositionEmbeddingSine (position_encoding.py:48-65),
    on even, ragged and non-rectangular masks; then the encoder half with the embedding derived on the device."""
    from salience_detr_b200.synthetic import build_model, make_inputs, sine_position_embedding
    model = build_model(layers=2).to(DEV)
    pe = pkg.PositionEmbeddingSine(128, temperature=10000, normalize=True, offset=-0.5)
    model.attach_position_embedding(pe)
    cpu_model = build_model(layers=2)
    for config in ("cpu_512", "resnet50_800_1333_bs2", "resnet50_800_1333_bs2_ragged", "resnet50_5scale_bs2", "holes"):
        if config == "holes":  # arbitrary (non-rectangular) padding: the scans must be true cumulative sums
            feats, masks, pos = make_inputs("resnet50_800_1333_bs2_ragged")
            g = torch.Generator().manual_seed(3)
            masks = [m | (torch.rand(m.shape, generator=g) < 0.2) for m in masks]
            masks = [m & ~torch.zeros_like(m).index_fill_(2, torch.tensor([0]), True) & ~torch.zeros_like(m).index_fill_(1, torch.tensor([0]), True)
                     for m in masks]  # keep the first row / column valid (non-zero valid sizes)
            pos = [sine_position_embedding(m, 128) for m in masks]
        else:
            feats, masks, pos = make_inputs(config)
        want = cpu_model.make_plan(masks)
        got = model.make_plan([m.to(DEV) for m in masks])
        assert got.level_token_nums == want.level_token_nums and got.focus_host == want.focus_host
        assert got.layer_num_query == want.layer_num_query and got.num_selected == want.num_selected
        assert torch.equal(got.focus_token_nums.cpu(), want.focus_token_nums)
        assert torch.equal(got.valid_ratios.cpu(), want.valid_ratios)
        assert torch.equal(got.keep.cpu(), want.keep)
        tok = model.position_tokens(got)
        ref = torch.cat([p.flatten(2) for p in pos], 2).transpose(1, 2)
        assert (tok.cpu() - ref).abs().max() < 3e-6, config
        m0 = masks[0].to(DEV)  # the module's reference-signature forward
        assert (pe(m0).cpu() - pos[0]).abs().max() < 3e-6
    feats, masks, pos = make_inputs("cpu_512", seed=2, device=DEV)
    with torch.no_grad():
        a, _ = model.forward_encoder(feats, masks, pos)
        b2, _ = model.forward_encoder(feats, masks, None)
    assert (a - b2).abs().max() < 2e-5


# ---- the benched callable at the benched configuration --------------------------------------------------------------------
FULL_CFG = dict(heads=8, points=4, topk_sa=300, num_layers=6, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
                layer_filter_ratio=(1.0, 0.8, 0.6, 0.6, 0.4, 0.2))


@pytest.mark.parametrize("config", ["resnet50_800_1333_bs2", "resnet50_800_1333_bs2_ragged"])
def test_config2_whole_path_benched_callable(pkg, config):
    """BASELINE.json configs[1] (800x1333, bs=2, Nv=22323, K=11363; even and ragged padding) through the callable that
    bench.py times -- ``EncoderRunner`` (one CUDA graph, ``gemm.MODE="auto"``, spatial tile order) -- against the CPU oracle
    (reference semantics salience_transformer.py:106-183): raw salience scores, selected-set overlap, the selection
    kernel bit-exact on the GPU's own scores, and -- with the oracle's indices injected, so both sides process the same
    tokens -- the encoder memory within the north-star tolerance (1e-3 abs).  The strict cuBLAS-fp32 mode is checked at
    the same size."""
    from salience_detr_b200.runner import EncoderRunner
    from salience_detr_b200.synthetic import build_model, make_inputs
    model = build_model().to(DEV)
    feats, masks, pos = make_inputs(config, device=DEV)
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    omem, ofilt = orc.encoder_half_forward(sd, [f.cpu() for f in feats], [m.cpu() for m in masks], [p.cpu() for p in pos],
                                           FULL_CFG, core="c", use_c_helpers=True)
    K = 11363
    assert ofilt["selected_inds"].shape == (2, K)
    assert ofilt["layer_num_query"] == [11363, 9090, 6817, 6817, 4545, 2272]
    oinds, ofg = ofilt["selected_inds"].to(DEV), ofilt["foreground_score"].to(DEV)
    focus = ofilt["focus_token_nums"].tolist() if "focus_token_nums" in ofilt else None
    assert pkg.gemm.MODE == "auto"
    runner = EncoderRunner(model, feats, masks, pos, use_graph=True, use_order=True)
    assert runner.graph is not None
    got_graph = runner.step()   # asynchronous on the runner's stream
    torch.cuda.synchronize()
    got_graph = got_graph.clone()
    plan = runner.plan
    if focus is not None:
        assert plan.focus_host == [int(f) for f in focus]
    for mode, tol_score, max_swaps in (("auto", 3e-4, 40), ("fp32", 3e-5, 12)):
        pkg.gemm.MODE = mode
        with torch.no_grad():
            mem, aux = model.forward_encoder(feats, masks, pos, plan=plan, use_order=True)
        if mode == "auto":  # the graph replays exactly this eager forward
            assert torch.equal(mem, got_graph)
        assert plan.num_selected == K and plan.layer_num_query == ofilt["layer_num_query"]
        err = (aux["raw_score"].cpu() - ofilt["raw_score"]).abs().max().item()
        assert err < tol_score, (mode, err)
        # op-level bit-exactness at full size on real score distributions: the oracle's selection of the GPU's own scores
        wi, ws, wf = orc.c_salience_select(aux["raw_score"].cpu(), plan.mask_flat.cpu(), plan.level_start_index.cpu(),
                                           torch.tensor(plan.level_size), plan.level_token_nums)
        assert torch.equal(aux["selected_inds"].cpu(), wi) and torch.equal(aux["foreground_score"].cpu(), wf)
        for i in range(2):  # end to end, only near-ties at a level's budget boundary may swap (scores differ by round-off)
            n = min(plan.focus_host[i], K)
            got, want = set(aux["selected_inds"][i, :n].tolist()), set(ofilt["selected_inds"][i, :n].tolist())
            assert len(got & want) >= n - max_swaps, (mode, i, n - len(got & want))
        feat = pkg.flatten_levels(feats)
        lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, model.level_embeds)])
        with torch.no_grad():
            mem_inj = model.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat,
                                    spatial_shapes=plan.spatial_shapes, level_start_index=plan.level_start_index,
                                    valid_ratios=plan.valid_ratios, foreground_score=ofg,
                                    focus_token_nums=plan.focus_token_nums,
                                    foreground_inds=[oinds[:, :n] for n in plan.layer_num_query], multi_level_masks=masks)
        err = (mem_inj.cpu() - omem).abs().max().item()
        assert err < 1e-3, (mode, err)


def test_salience_targets_kernel_vs_reference_golden(pkg):
    """sdetr_salience_targets (one launch) against the reference SalienceCriterion's target maps, loss and gradient
    (tests/golden/salience_criterion.npz); an image without boxes; many boxes."""
    g, _ = load_golden("salience_criterion")
    shapes = [tuple(int(v) for v in r) for r in g["shapes"]]
    fg = [g[f"fg{i}"].to(DEV).requires_grad_(True) for i in range(4)]
    targets = [{"boxes": g["boxes0"].to(DEV)}, {"boxes": g["boxes1"].to(DEV)}]
    sizes = [tuple(int(v) for v in r) for r in g["image_sizes"]]
    strides = [tuple(float(v) for v in r) for r in g["strides"]]
    crit = pkg.SalienceCriterion()
    n0 = pkg.cabi.launch_count()
    mt = crit.mask_targets(shapes, targets, strides, sizes, torch.device(DEV))
    assert pkg.cabi.launch_count() == n0 + 1
    assert (mt.cpu() - g["mask_targets"]).abs().max() < 1e-6 and torch.equal(mt.cpu() > 0, g["mask_targets"] > 0)
    loss = crit(fg, targets, strides, sizes)["loss_salience"]
    assert abs(loss.item() - g["loss"].item()) < 1e-5
    loss.backward()
    for i in range(4):
        assert (fg[i].grad.cpu() - g[f"grad{i}"]).abs().max() < 1e-6
    gen = torch.Generator().manual_seed(5)
    many = torch.cat([torch.rand(150, 2, generator=gen) * 0.8 + 0.1, torch.rand(150, 2, generator=gen) * 0.4 + 0.01], -1)
    t2 = [{"boxes": torch.zeros(0, 4, device=DEV)}, {"boxes": many.to(DEV)}]
    a = crit.mask_targets(shapes, t2, strides, sizes, torch.device(DEV)).cpu()
    w = crit.mask_targets(shapes, [{"boxes": torch.zeros(0, 4)}, {"boxes": many}], strides, sizes, torch.device("cpu"))
    assert a[0].abs().max() == 0 and (a - w).abs().max() < 1e-6


def test_ffn_fused_layernorm(pkg):
    """Encoder FFN + LayerNorm (sdetr_ffn_fused_layernorm) against an fp64 reference and against the two-GEMM path: the full
    grid and grids capped at a few CTAs (many tiles per CTA), ragged last panel, strided input rows, bare-FFN mode, in-place
    output, bit-reproducible."""
    g = torch.Generator().manual_seed(11)
    F = torch.nn.functional
    lib = pkg.cabi.lib()
    try:
        for rows, hidden in [(128, 256), (1000, 2048), (22726, 2048), (19500, 1024), (300, 128), (4545, 2048)]:
            x = torch.randn(rows, 256, generator=g).to(DEV)
            w1 = (torch.randn(hidden, 256, generator=g) / 16).to(DEV)
            b1 = torch.randn(hidden, generator=g).to(DEV)
            w2 = (torch.randn(256, hidden, generator=g) / hidden ** 0.5).to(DEV)
            b2 = torch.randn(256, generator=g).to(DEV)
            gamma = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV)
            beta = (0.1 * torch.randn(256, generator=g)).to(DEV)
            s1, s2 = pkg.cabi.split_f16_pair(w1), pkg.cabi.split_f16_pair(w2)
            f64 = F.linear(F.relu(F.linear(x.double(), w1.double(), b1.double())), w2.double(), b2.double())
            ref = F.layer_norm(x.double() + f64, (256,), gamma.double(), beta.double(), 1e-5)
            two = pkg.cabi.gemm_f16x3_pre(pkg.cabi.gemm_f16x3_pre(x, *s1, b1, 0), *s2, b2, 1)
            e_two = (two.double() - f64).abs().max().item()
            for ctas in (0, 7, 97, 1):
                lib.sdetr_set_persistent_ctas(ctas)
                bare = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, b2)
                err = (bare.double() - f64).abs().max().item()
                assert err < 1e-4 and err < 4 * e_two + 1e-6, (rows, hidden, ctas, err, e_two)
                y = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, b2, gamma, beta, 1e-5)
                assert (y.double() - ref).abs().max().item() < 1e-4, (rows, hidden, ctas)
                assert torch.equal(pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, b2, gamma, beta, 1e-5), y)
            lib.sdetr_set_persistent_ctas(0)
            # in place (the layer's use) and strided input rows
            xin = x.clone()
            pkg.cabi.ffn_fused_layernorm(xin, s1, b1, s2, b2, gamma, beta, 1e-5, out=xin)
            assert (xin.double() - ref).abs().max().item() < 1e-4
            wide = torch.zeros(rows, 320, device=DEV)
            wide[:, :256] = x
            ys = pkg.cabi.ffn_fused_layernorm(wide[:, :256], s1, b1, s2, b2, gamma, beta, 1e-5)
            assert (ys.double() - ref).abs().max().item() < 1e-4
        # the documented value domain: large activations, six decades inside a row
        x = (torch.randn(700, 256, generator=g) * torch.logspace(-3, 2, 256)).to(DEV)
        f64 = F.linear(F.relu(F.linear(x.double(), w1.double(), b1.double())), w2.double(), b2.double())
        bare = pkg.cabi.ffn_fused_layernorm(x, s1, b1, s2, b2)
        assert ((bare.double() - f64).abs().max() / f64.abs().max()).item() < 2e-6
    finally:
        lib.sdetr_set_persistent_ctas(0)


def test_mask_predictor_level(pkg):
    """Score modulation + MaskPredictor of a small level as two launches (sdetr_mask_predictor_level) against the module's own
    torch forward on the modulated tokens (reference :16-47, :134-143) in fp64; ragged last tile, with / without a coarser level,
    bit-reproducible."""
    g = torch.Generator().manual_seed(21)
    F = torch.nn.functional
    mp = pkg.salience_transformer.MaskPredictor(256, 256)
    with torch.no_grad():
        for p_ in mp.parameters():
            p_.copy_(torch.randn(p_.shape, generator=g) * (0.08 if p_.dim() > 1 else 0.2) + (1.0 if p_.dim() == 1 and p_.numel() == 256 and p_ is mp.layer1[0].weight else 0.0))
    mp64 = __import__("copy").deepcopy(mp).double()
    mp = mp.to(DEV)
    alpha = torch.tensor([0.3, -0.2, 0.7], device=DEV)
    for b, (h, w), (hc, wc) in [(2, (13, 21), (0, 0)), (2, (25, 42), (13, 21)), (3, (7, 9), (4, 5)), (1, (1, 5), (1, 3)), (2, (50, 84), (25, 42))]:
        lead, tail = 37, 11
        nv = lead + h * w + hc * wc + tail
        mem = torch.randn(b, nv, 256, generator=g).to(DEV)
        raw = torch.zeros(b, nv, device=DEV)
        coarse = None
        if hc:
            raw[:, lead + h * w:lead + h * w + hc * wc] = torch.randn(b, hc * wc, generator=g).to(DEV)
            coarse = raw[:, lead + h * w:lead + h * w + hc * wc]
        ln = mp.layer1[0]
        keep = raw.clone()
        pkg.cabi.mask_predictor_level(mem, lead, h, w, coarse, hc, wc, alpha, 1, ln.weight, ln.bias, ln.eps, *mp.transposed_weights(), raw, lead)
        m = mem[:, lead:lead + h * w].double().cpu()
        if hc:
            up = F.interpolate(coarse.double().cpu().reshape(b, 1, hc, wc), size=(h, w), mode="bilinear", align_corners=True)
            m = m + m * up.view(b, 1, h * w).transpose(1, 2) * float(alpha[1])
        with torch.no_grad():
            want = mp64(m).squeeze(-1)
        got = raw[:, lead:lead + h * w]
        assert (got.double().cpu() - want).abs().max().item() < 3e-5, (b, h, w)
        outside = torch.ones(nv, dtype=torch.bool)
        outside[lead:lead + h * w] = False
        assert torch.equal(raw[:, outside], keep[:, outside])  # nothing but the level's slice is written
        again = keep.clone()
        pkg.cabi.mask_predictor_level(mem, lead, h, w, again[:, lead + h * w:lead + h * w + hc * wc] if hc else None, hc, wc, alpha, 1,
                                      ln.weight, ln.bias, ln.eps, *mp.transposed_weights(), again, lead)
        assert torch.equal(again, raw)


def test_linear_train_tensor_core(pkg):
    """Training-path Linear on the 3xFP16 kernel (forward and input gradient with DEVICE-side power-of-two scales; weight gradient on
    cuBLAS) against fp64 autograd: activations O(1), gradients of 1e-8 .. 1e+3 (far outside the fixed range of the inference entry
    point), ragged N, bias / no bias, non-contiguous upstream gradient; pow2_scale itself; fallback shapes."""
    g = torch.Generator().manual_seed(31)
    F = torch.nn.functional
    for n, tgt in [(1000, 12), (70001, 14), (3, 0)]:
        x = (torch.randn(n, generator=g) * 10.0 ** float(torch.randint(-9, 4, (1,), generator=g))).to(DEV)
        s = pkg.cabi.pow2_scale(x, tgt).item()
        amax = x.abs().max().item()
        assert 2.0 ** (tgt - 1) <= amax * s < 2.0 ** tgt and s == 2.0 ** round(__import__("math").log2(s))
    assert pkg.cabi.pow2_scale(torch.zeros(100, device=DEV), 12).item() == 1.0
    for rows, k, n, gscale, bias in [(3000, 256, 2048, 1e-7, True), (5000, 2048, 256, 3e2, True), (2500, 256, 384, 1e-3, False),
                                     (4097, 64, 91, 1.0, True), (2400, 128, 64, 1e-5, True)]:
        x = torch.randn(rows, k, generator=g).to(DEV).requires_grad_(True)
        w = (torch.randn(n, k, generator=g) / k ** 0.5).to(DEV).requires_grad_(True)
        b = torch.randn(n, generator=g).to(DEV).requires_grad_(True) if bias else None
        dy = (torch.randn(n, rows, generator=g) * gscale).to(DEV).t()  # non-contiguous upstream gradient
        y = pkg.gemm.linear_train(x, w, b)
        assert y.grad_fn is not None and "LinearF16x3" in type(y.grad_fn).__name__
        y.backward(dy)
        x64, w64 = x.detach().double().requires_grad_(True), w.detach().double().requires_grad_(True)
        b64 = b.detach().double().requires_grad_(True) if bias else None
        y64 = F.linear(x64, w64, b64)
        y64.backward(dy.double())
        assert (y.detach().double() - y64.detach()).abs().max().item() < 2e-5 * y64.detach().abs().max().item()
        for got, want in [(x.grad, x64.grad), (w.grad, w64.grad)] + ([(b.grad, b64.grad)] if bias else []):
            err = (got.double() - want).abs().max().item()
            assert err <= 3e-5 * want.abs().max().item(), (rows, k, n, gscale, err, want.abs().max().item())
    # shapes the kernel does not take fall back to F.linear: few rows, K not a multiple of 64
    for rows, k in [(100, 256), (5000, 100)]:
        x = torch.randn(rows, k, device=DEV, requires_grad=True)
        w = torch.randn(32, k, device=DEV, requires_grad=True)
        y = pkg.gemm.linear_train(x, w, None)
        assert "LinearF16x3" not in type(y.grad_fn).__name__
    # the context manager routes nn.Linear through it and restores F.linear afterwards
    lin = torch.nn.Linear(256, 512).to(DEV)
    xin = torch.randn(4000, 256, device=DEV)
    with pkg.gemm.tensor_core_linears():
        out = lin(xin)
    assert "LinearF16x3" in type(out.grad_fn).__name__ and torch.nn.functional.linear is pkg.gemm._orig_linear
    assert (out - F.linear(xin, lin.weight, lin.bias)).abs().max().item() < 3e-5
    torch.relu_(out)  # the Function's output is not a view: in-place ops on it are legal (the FFN's ReLU(inplace=True))
