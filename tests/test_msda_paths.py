"""Multi-scale deformable attention on every forward and backward kernel path, against a float64 reference.

`msda_forward_dispatch` (csrc/msda_forward.cu) picks among six kernel families; `predict_path` restates its rule:
  F1 msda_fwd_tma_kernel      D=32/L=4/P=4, schedule 1, option msda_tma=1, a query order, aligned inputs
  F2 msda_fwd_w32_kernel      the same shape, schedule 1, option msda_warp_per_item 1 or 2
  F3 msda_fwd_kernel<32,4,4,..,SMEM_BCAST=true,THREADS>   the default at D=32/L=4/P=4 (THREADS from msda_threads under
                                                          schedule 1)
  F4 msda_fwd_kernel<32,4,4,..,MINB,false>                option msda_smem_broadcast=0 (MINB from msda_min_blocks)
  F5 msda_fwd_kernel<32,5,4> and <64,4,4>
  F6 msda_fwd_generic_kernel  every other shape, and D=32/L=4/P=4 when loc/attn are not 16-byte aligned or the fused
                              projection's row stride is not a multiple of 4
Each runs plain (sampling locations and weights given) or fused (softmax and location arithmetic in the kernel, from 2-d
reference points or 4-d reference boxes).  The backward has one template instance per head dim in {4, ..., 128}, with
float atomics or with the fixed-point deterministic accumulation.

One case of every distinct dispatch input runs under torch.profiler (in a child process), which checks that the
predicted kernel ran; the kernel depends on nothing else, so this confirms the kernel of every case.  Results are compared with
`msda_ref`, a float64 restatement of the reference kernel's arithmetic (ms_deform_im2col_cuda.cuh:22-73, 226-288), under
element-wise bounds built from the same reference run on absolute values: the error of a float32 sum of products is
bounded by a multiple of 2^-24 times the sum of the absolute products, whatever the sign pattern.  Inputs splice
adversarial sampling locations into random ones: exact pixel centres, coordinates 0 and 1, h_im exactly -1 and exactly H
and one ulp inside each, far outside, NaN and +-inf, on 1x1, 1xW and Hx1 levels."""
import json
import math
import os
import subprocess
import sys
import time
import zlib

import pytest
import torch

from oracle import oracle as orc

DEV = "cuda:0"
U = 2.0 ** -24  # unit round-off of float32
TINY = 2.0 ** -140  # absolute slack for subnormal products (gradients scaled to 1e-30)
DEFAULTS = {"msda_tma": 0, "msda_warp_per_item": 0, "msda_threads": 256, "msda_chunk": 64, "msda_smem_broadcast": 1,
            "msda_min_blocks": 4}

# Bound constants c of |got - ref| <= c * 2^-24 * S + TINY, S the same sum over absolute values.  Each is about four
# times the largest c observed over every case of this file on an H100 80GB HBM3 at 700 W (noted beside it).
C_FWD = 50.0   # forward output, every path (observed 12.7, F3)
C_LOC = 8.0    # fused loc_out against fused_ref (observed 1.9)
C_ATTN = 3.0   # fused attn_out, times the __expf / sum / reciprocal error model in test_forward_path (observed 0.69)
C_GV = 20.0    # grad_value, float atomics and fixed point, 16384 contributions per element included (observed 5.2)
C_GA = 12.0    # grad_attn (observed 3.0, 4096 queries on one 2x2 neighbourhood)
C_GL = 10.0    # grad_loc (observed 2.4)
FLT_MIN = 2.0 ** -126  # red.global.add.f32 flushes subnormal inputs and results to zero: up to this much per addition


# ---- the float64 reference ---------------------------------------------------------------------------------------------
def msda_ref(value, shapes, loc, attn, f32_coords=True, unit=False):
    """value (b,Nv,M,D), loc (b,Nq,M,L,P,2), attn (b,Nq,M,L,P) -> (b,Nq,M*D), in float64.

    The arithmetic of the reference kernel: h_im = y*H - 0.5, w_im = x*W - 0.5; a point counts only when
    h_im > -1, w_im > -1, h_im < H and w_im < W; the corners come from floor and a corner outside the map contributes 0; a
    non-finite location contributes 0.  With `f32_coords` h_im and w_im are rounded to float32 once, as the kernels'
    fmaf(y, H, -0.5f) does (y*H - 0.5 is exact in float64 for float32 y), so that every in/out and floor decision is the
    kernels' own.  The fractions come from floor of a detached h_im, so autograd through `loc` gives the kernels'
    one-sided derivative at integer h_im.  `unit` weights every valid corner by 1 instead of its bilinear weight (the
    scale of the location gradient's bound)."""
    b, _, M, D = value.shape
    nq, L, P = loc.shape[1], loc.shape[3], loc.shape[4]
    value, loc, attn = value.double(), loc.double(), attn.double()
    out = value.new_zeros(b, nq, M, D)
    bi = torch.arange(b, device=value.device).view(b, 1, 1, 1)
    mi = torch.arange(M, device=value.device).view(1, 1, M, 1)
    start = 0
    for l, (H, W) in enumerate(shapes):
        x, y = loc[:, :, :, l, :, 0], loc[:, :, :, l, :, 1]  # (b, nq, M, P)
        finite = torch.isfinite(x) & torch.isfinite(y)
        x, y = torch.where(finite, x, 0.0), torch.where(finite, y, 0.0)
        h_im, w_im = y * H - 0.5, x * W - 0.5
        if f32_coords:
            h_im, w_im = h_im.float().double(), w_im.float().double()
        inside = finite & (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
        h_im, w_im = torch.where(inside, h_im, 0.0), torch.where(inside, w_im, 0.0)
        h0, w0 = torch.floor(h_im.detach()), torch.floor(w_im.detach())
        ly, lx = h_im - h0, w_im - w0
        hy, hx = 1 - ly, 1 - lx
        y0, x0 = h0.long(), w0.long()
        v_l = value[:, start:start + H * W]
        a = attn[:, :, :, l]
        for dy, dx, wgt in ((0, 0, hy * hx), (0, 1, hy * lx), (1, 0, ly * hx), (1, 1, ly * lx)):
            yy, xx = y0 + dy, x0 + dx
            ok = inside & (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            idx = yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)
            w = torch.where(ok, (torch.ones_like(wgt) if unit else wgt) * a, 0.0)
            out = out + (w[..., None] * v_l[bi, idx, mi]).sum(3)
        start += H * W
    return out.reshape(b, nq, M * D)


def fused_ref(ref_points, proj, shapes, M, L, P):
    """Softmax and sampling locations from the fused projection (ms_deform_attn.py:170-176), in float64.
    proj (b,Nq,>=3n), n = M*L*P: offsets (M,L,P,2) of every head, then logits (M,L*P).  -> (loc, attn, logit - max)."""
    b, nq = proj.shape[:2]
    n = M * L * P
    proj, ref = proj.double(), ref_points.double()
    off = proj[..., :2 * n].reshape(b, nq, M, L, P, 2)
    logit = proj[..., 2 * n:3 * n].reshape(b, nq, M, L * P)
    shifted = logit - logit.max(-1, keepdim=True)[0]
    attn = shifted.softmax(-1).view(b, nq, M, L, P)
    if ref.shape[-1] == 2:
        norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
        loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    else:
        loc = ref[:, :, None, :, None, :2] + off / P * ref[:, :, None, :, None, 2:] * 0.5
    return loc, attn, shifted.view(b, nq, M, L, P)


def forward_scale(value, shapes, loc, attn):
    """S of the forward bound: the reference on |value| and |attn|."""
    return msda_ref(value.abs(), shapes, loc, attn.abs())


def backward_scales(value, shapes, loc, attn, gout):
    """S of the three gradient bounds: grad_value on |attn|, |grad_out|; grad_attn as the sum of |w * go * v|; grad_loc
    as W*|a| (x) and H*|a| (y) times the sum of |go * v| over the valid corners."""
    va, aa, ga = value.double().abs(), attn.double().abs(), gout.double().abs()
    v = va.clone().requires_grad_(True)
    (msda_ref(v, shapes, loc, aa) * ga).sum().backward()
    a = aa.clone().requires_grad_(True)
    (msda_ref(va, shapes, loc, a) * ga).sum().backward()
    one = torch.ones_like(aa, requires_grad=True)
    (msda_ref(va, shapes, loc, one, unit=True) * ga).sum().backward()
    hw = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
    s_loc = (aa * one.grad)[..., None] * hw[None, None, None, :, None, :]
    return v.grad, a.grad, s_loc


def reference_grads(value, shapes, loc, attn, gout):
    v, l, a = (t.double().clone().requires_grad_(True) for t in (value, loc, attn))
    (msda_ref(v, shapes, l, a) * gout.double()).sum().backward()
    return v.grad, l.grad, a.grad


def within(got, want, scale, c, tiny=TINY):
    """Largest |got - want| / (c * U * scale + tiny); <= 1 passes.  NaN anywhere fails."""
    err = (got.double().cpu() - want).abs()
    ratio = err / (c * U * scale + tiny)
    return float(ratio.max()) if ratio.numel() else 0.0


# ---- inputs ------------------------------------------------------------------------------------------------------------
def level_geometry(shapes):
    st = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
    return st, lsi, int(st.prod(1).sum())


def edge_coords(S):
    """Coordinates (float32) of the edges of a level of size S (a power of two, so y*S is exact): pixel centres, 0 and 1,
    h_im = -1 and one ulp inside, h_im = S and one ulp inside, far outside and non-finite."""
    c = [(i + 0.5) / S for i in range(S)] + [0.0, 1.0, -0.5 / S, -(0.5 - 2.0 ** -24) / S, (S + 0.5) / S,
                                              1.0 + 0.5 / S - 2.0 ** -23, -1e3, 1e3, 3e38, float("nan"),
                                              float("inf"), -float("inf")]
    return torch.tensor(c, dtype=torch.float32)


def splice_edges(loc, shapes, g, frac=0.35):
    """Replace about `frac` of the coordinates of loc (..., L, P, 2) by edge coordinates of their level, in place."""
    for l, (H, W) in enumerate(shapes):
        for k, S in ((0, W), (1, H)):
            c = loc[..., l, :, k]
            pick = torch.rand(c.shape, generator=g) < frac
            e = edge_coords(S)
            c[pick] = e[torch.randint(0, len(e), c.shape, generator=g)][pick]


def make_plain(b, shapes, M, D, P, nq, g, spread="wide"):
    L = len(shapes)
    _, _, nv = level_geometry(shapes)
    value = torch.randn(b, nv, M, D, generator=g)
    if spread == "local":  # every query within a pixel or two of the map centre: inside the TMA windows
        loc = 0.5 + torch.randn(b, nq, M, L, P, 2, generator=g) * 0.02
    else:
        loc = torch.rand(b, nq, M, L, P, 2, generator=g) * 1.2 - 0.1
        splice_edges(loc, shapes, g)
    attn = torch.randn(b, nq, M, L, P, generator=g)
    return value, loc, attn


def make_fused(b, shapes, M, D, P, nq, g, ref_dim, spread="wide"):
    """(value, ref, proj): offsets of a few pixels, logits of spread 2; a third of the reference points sit on edge
    coordinates with zero offsets for a third of their points, so that loc equals the edge coordinate exactly."""
    L = len(shapes)
    _, _, nv = level_geometry(shapes)
    n = M * L * P
    value = torch.randn(b, nv, M, D, generator=g)
    proj = torch.randn(b, nq, 3 * n, generator=g) * 2
    if spread == "local":
        ref = torch.full((b, nq, L, 2), 0.5) + torch.randn(b, nq, L, 2, generator=g) * 0.01
        proj[..., :2 * n] *= 0.2
    else:
        ref = torch.rand(b, nq, L, 2, generator=g) * 1.2 - 0.1
        off = proj[..., :2 * n].view(b, nq, M, L, P, 2)
        off[torch.rand(b, nq, M, L, P, generator=g) < 0.35] = 0.0
        for l, (H, W) in enumerate(shapes):
            for k, S in ((0, W), (1, H)):
                pick = torch.rand(b, nq, generator=g) < 0.35
                e = edge_coords(S)
                ref[..., l, k][pick] = e[torch.randint(0, len(e), (b, nq), generator=g)][pick]
    if ref_dim == 4:
        ref = torch.cat([ref, torch.rand(b, nq, L, 2, generator=g) * 0.5], -1)
    return value, ref.contiguous(), proj


# ---- the host's path rule ----------------------------------------------------------------------------------------------
def predict_path(D, L, P, schedule, fused, aligned, options, ordered):
    """(family, kernel name as the profiler shows it) that msda_forward_dispatch launches."""
    tf = lambda v: "true" if v else "false"  # noqa: E731
    F, HM = tf(fused), tf(schedule == 1)
    prod = aligned and (D, L, P) == (32, 4, 4)
    if prod and schedule == 1 and options["msda_tma"] and ordered:
        return "F1", f"msda_fwd_tma_kernel<{F}>"
    if prod and schedule == 1 and options["msda_warp_per_item"]:
        k = options["msda_warp_per_item"]
        return "F2", f"msda_fwd_w32_kernel<{F}, {k}, {4 if k == 2 else 6}>"
    if prod and options["msda_smem_broadcast"]:
        threads = options["msda_threads"] if schedule == 1 else 256
        return "F3", f"msda_fwd_kernel<32, 4, 4, {F}, {HM}, {256 * 4 // threads}, true, {threads}>"
    if prod:
        return "F4", f"msda_fwd_kernel<32, 4, 4, {F}, {HM}, {options['msda_min_blocks']}, false, 256>"
    if aligned and (D, L, P) in ((32, 5, 4), (64, 4, 4)):
        return "F5", f"msda_fwd_kernel<{D}, {L}, {P}, {F}, {HM}, 2, false, 256>"
    return "F6", "msda_fwd_generic_kernel"


def dispatch_key(c):
    """Everything msda_forward_dispatch decides on: two cases with the same key launch the same kernel."""
    return (c["D"], len(c["shapes"]), c["P"], c["sched"], c["kind"] != "plain", not c["misalign"],
            tuple(sorted({**DEFAULTS, **c["opts"]}.items())), c["order"])


def predict_case(c):
    D, L, P, sched, fused, aligned, opts, ordered = dispatch_key(c)
    return predict_path(D, L, P, sched, fused, aligned, dict(opts), ordered)


# ---- forward cases -----------------------------------------------------------------------------------------------------
PROD = [(32, 64), (16, 32), (8, 16), (4, 8)]  # powers of two (exact edges), W != H (x and y distinguishable)
KINDS = ("plain", "fused2", "fused4")


def fcase(id, b, shapes, M, D, P, nq, sched=(0, 1), opts=None, order=False, misalign=False, strided=True,
          spread="wide", kinds=KINDS):
    return [dict(id=f"{id}-{k}-s{s}", b=b, shapes=shapes, M=M, D=D, P=P, nq=nq, sched=s, kind=k, opts=opts or {},
                 order=order, misalign=misalign, strided=strided, spread=spread) for k in kinds for s in sched]


FWD = [
    *fcase("F3", 2, PROD, 8, 32, 4, 777),
    *fcase("F3_ordered", 2, PROD, 8, 32, 4, 777, order=True),
    *fcase("F3_contiguous", 1, PROD, 8, 32, 4, 65, strided=False),
    *[c for t in (256, 512, 1024) for ch in (8, 64, 100, 4096)
      for c in fcase(f"F3_t{t}_c{ch}", 2, PROD, 3, 32, 4, 777, sched=(1,), order=True,
                     opts={"msda_threads": t, "msda_chunk": ch})],
    *[c for mb in (2, 3, 4, 5, 6)
      for c in fcase(f"F4_minb{mb}", 2, PROD, 3, 32, 4, 129, order=True,
                     opts={"msda_smem_broadcast": 0, "msda_min_blocks": mb})],
    *[c for k in (1, 2) for o in (False, True)
      for c in fcase(f"F2_w{k}{'_ordered' if o else ''}", 2, PROD, 8, 32, 4, 777, sched=(1,), order=o,
                     opts={"msda_warp_per_item": k})],
    *fcase("F2_chunk100", 1, PROD, 3, 32, 4, 777, sched=(1,), opts={"msda_warp_per_item": 2, "msda_chunk": 100}),
    *fcase("F1_wide", 2, PROD, 8, 32, 4, 777, sched=(1,), order=True, opts={"msda_tma": 1}),
    *fcase("F1_local", 2, PROD, 8, 32, 4, 777, sched=(1,), order=True, opts={"msda_tma": 1}, spread="local"),
    *fcase("F1_chunk8", 1, [(40, 56), (20, 28), (10, 14), (5, 7)], 2, 32, 4, 333, sched=(1,), order=True,
           opts={"msda_tma": 1, "msda_chunk": 8}),
    *fcase("F1_unordered", 1, PROD, 2, 32, 4, 65, sched=(1,), opts={"msda_tma": 1}),  # no order: not F1
    *fcase("F5_L5", 2, [(16, 32), (8, 16), (4, 8), (1, 8), (8, 1)], 3, 32, 4, 65),
    *fcase("F5_D64", 3, [(8, 16), (1, 1), (16, 1), (4, 4)], 3, 64, 4, 63, order=True),
    *fcase("F6_misaligned", 2, PROD, 8, 32, 4, 777, misalign=True, order=True),
    *fcase("F6_misaligned_tma", 1, PROD, 8, 32, 4, 65, sched=(1,), misalign=True, order=True, opts={"msda_tma": 1}),
    *fcase("F6_misaligned_w32", 1, PROD, 8, 32, 4, 65, sched=(1,), misalign=True, opts={"msda_warp_per_item": 1}),
    *fcase("F6_D4_L1_P1", 1, [(8, 16)], 1, 4, 1, 1, sched=(0,)),
    *fcase("F6_D8_L3_P2", 3, [(16, 8), (1, 1), (8, 1)], 3, 8, 2, 63, sched=(0,), order=True),
    *fcase("F6_D16_L8_P8", 2, [(16, 16), (8, 8), (1, 8), (4, 4), (8, 1), (2, 2), (1, 1), (2, 4)], 1, 16, 8, 65),
    *fcase("F6_D128_L3_P2", 1, [(16, 32), (8, 16), (4, 8)], 3, 128, 2, 777, sched=(1,), order=True),
    *fcase("F6_D256_L1_P8", 2, [(8, 16)], 1, 256, 8, 65, sched=(0,)),
    *fcase("F6_D32_P8", 1, PROD, 3, 32, 8, 65, sched=(1,), strided=False),
]


# ---- CPU: the reference against independent ones ---------------------------------------------------------------------
def _plain_inputs(seed, shapes=((8, 16), (4, 8), (1, 4), (2, 1)), b=2, M=3, D=8, P=3, nq=17):
    g = torch.Generator().manual_seed(seed)
    return make_plain(b, list(shapes), M, D, P, nq, g)


def test_ref_matches_grid_sample():
    """Away from the edges msda_ref equals the reference's PyTorch path (grid_sample, oracle.msda_core_torch)."""
    g = torch.Generator().manual_seed(1)
    shapes = [(7, 9), (4, 5), (2, 3)]
    _, _, nv = level_geometry(shapes)
    value = torch.randn(2, nv, 3, 8, generator=g, dtype=torch.float64)
    loc = torch.rand(2, 11, 3, 3, 2, 2, generator=g, dtype=torch.float64) * 0.9 + 0.05
    attn = torch.randn(2, 11, 3, 3, 2, generator=g, dtype=torch.float64)
    want = orc.msda_core_torch(value, shapes, loc, attn)
    got = msda_ref(value, shapes, loc, attn, f32_coords=False)
    assert (got - want).abs().max() < 1e-12


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_ref_matches_c_oracle_at_edges(seed):
    """msda_ref agrees with the C oracle (float32) to its round-off, edge locations included: forward and all three
    gradients.  The oracle sums L*P products per output in float32, so its error is below (L*P + 4) u S."""
    shapes = [(8, 16), (4, 8), (1, 4), (2, 1)]
    value, loc, attn = _plain_inputs(seed, shapes)
    st, lsi, _ = level_geometry(shapes)
    L, P = loc.shape[3], loc.shape[4]
    c = L * P + 4
    want = orc.c_msda_forward(value, st, lsi, loc, attn)
    assert within(want, msda_ref(value, shapes, loc, attn), forward_scale(value, shapes, loc, attn), c) <= 1
    gout = torch.randn(want.shape, generator=torch.Generator().manual_seed(seed + 10))
    wv, wl, wa = orc.c_msda_backward(value, st, lsi, loc, attn, gout)
    rv, rl, ra = reference_grads(value, shapes, loc, attn, gout)
    sv, sa, sl = backward_scales(value, shapes, loc, attn, gout)
    nq = loc.shape[1]
    assert within(wv, rv, sv, nq * P + 4) <= 1
    assert within(wa, ra, sa, 4 * value.shape[-1]) <= 1
    assert within(wl, rl, sl, 4 * value.shape[-1]) <= 1


def test_ref_location_gradient_matches_finite_difference():
    """Autograd through msda_ref's location equals a central finite difference where the sample is off pixel centres."""
    g = torch.Generator().manual_seed(3)
    shapes = [(6, 7), (3, 4)]
    _, _, nv = level_geometry(shapes)
    value = torch.randn(1, nv, 2, 4, generator=g, dtype=torch.float64)
    loc = torch.rand(1, 5, 2, 2, 2, 2, generator=g, dtype=torch.float64) * 0.8 + 0.1
    attn = torch.randn(1, 5, 2, 2, 2, generator=g, dtype=torch.float64)
    for l, (H, W) in enumerate(shapes):  # keep h_im, w_im at least 0.05 from an integer
        for k, S in ((0, W), (1, H)):
            c = loc[..., l, :, k] * S - 0.5
            fr = c - c.floor()
            loc[..., l, :, k] = (c.floor() + fr.clamp(0.05, 0.95) + 0.5) / S
    gout = torch.randn(1, 5, 8, generator=g, dtype=torch.float64)
    lg = loc.clone().requires_grad_(True)
    (msda_ref(value, shapes, lg, attn, f32_coords=False) * gout).sum().backward()
    h = 1e-7
    fd = torch.zeros_like(loc)
    flat = loc.view(-1)
    for i in range(flat.numel()):
        p, m = loc.clone(), loc.clone()
        p.view(-1)[i] += h
        m.view(-1)[i] -= h
        fd.view(-1)[i] = ((msda_ref(value, shapes, p, attn, f32_coords=False) -
                           msda_ref(value, shapes, m, attn, f32_coords=False)) * gout).sum() / (2 * h)
    assert (lg.grad - fd).abs().max() <= 1e-6 * max(1.0, fd.abs().max().item())


def test_case_table_reaches_every_path():
    """The forward table predicts every family F1-F6, each plain, fused 2-d and fused 4-d."""
    got = {(predict_path(c["D"], len(c["shapes"]), c["P"], c["sched"], c["kind"] != "plain", not c["misalign"],
                         {**DEFAULTS, **c["opts"]}, c["order"])[0], c["kind"]) for c in FWD}
    assert got == {(f, k) for f in ("F1", "F2", "F3", "F4", "F5", "F6") for k in KINDS}


def test_predict_path_names():
    opts = dict(DEFAULTS)
    assert predict_path(32, 4, 4, 1, True, True, opts, True) == ("F3", "msda_fwd_kernel<32, 4, 4, true, true, 4, true, 256>")
    assert predict_path(32, 4, 4, 1, True, True, {**opts, "msda_threads": 512}, True)[1].endswith("2, true, 512>")
    assert predict_path(32, 4, 4, 1, False, True, {**opts, "msda_tma": 1}, False)[0] == "F3"
    assert predict_path(32, 4, 4, 0, False, True, {**opts, "msda_warp_per_item": 2}, True)[0] == "F3"
    assert predict_path(32, 4, 4, 1, False, False, {**opts, "msda_tma": 1}, True)[0] == "F6"


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


@pytest.fixture(autouse=True)
def _restore_options(request):
    """The library options are process-global and have no getter: every test leaves them at the shipped defaults."""
    yield
    if "pkg" in request.fixturenames:
        cabi = request.getfixturevalue("pkg").cabi
        for k, v in DEFAULTS.items():
            cabi.set_option(k, v)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def value_buffer(value, strided):
    """(buffer, batch stride, token stride, offset) holding value (b,Nv,M,D).  Strided: a wide buffer of 6*M*D + 4 floats
    per token, three unused rows between images and the slice at a 16-byte aligned column offset; every float outside
    the slice is NaN, so a stray read shows up in the output."""
    b, nv, M, D = value.shape
    if not strided:
        return value.to(DEV).contiguous(), nv * M * D, M * D, 0
    ts, off, gap = 6 * M * D + 4, 2 * M * D + 4, 3
    buf = torch.full((b, nv + gap, ts), float("nan"), device=DEV)
    buf[:, :nv, off:off + M * D] = value.view(b, nv, M * D).to(DEV)
    return buf, (nv + gap) * ts, ts, off


def misaligned(t):
    """A copy of t whose data pointer is 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 1, device=DEV)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


def forward_plain(pkg, vb, shapes_d, lsi_d, loc, attn, M, D, L, P, nv, order, sched):
    buf, bs, ts, off = vb
    b, nq = loc.shape[:2]
    out = torch.empty(b, nq, M * D, device=DEV)
    rc = pkg.cabi.lib().sdetr_msda_forward_ex(buf.data_ptr() + 4 * off, bs, ts, shapes_d.data_ptr(), lsi_d.data_ptr(),
                                               loc.data_ptr(), attn.data_ptr(), out.data_ptr(), b, nv, M, D, L, nq, P,
                                               _ptr(order), sched, pkg.cabi._stream())
    pkg.cabi._check(rc, "sdetr_msda_forward_ex")
    return out


def random_orders(b, nq, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.stack([torch.randperm(nq, generator=g) for _ in range(b)]).to(torch.int32).to(DEV) for _ in range(2)]


def setup_forward(pkg, c):
    """Set the case's options and build its inputs on the device -> (run(order), order, orders, host inputs)."""
    b, shapes, M, D, P, nq, sched, kind = c["b"], c["shapes"], c["M"], c["D"], c["P"], c["nq"], c["sched"], c["kind"]
    L = len(shapes)
    for k, v in {**DEFAULTS, **c["opts"]}.items():
        pkg.cabi.set_option(k, v)
    pkg.cabi.msda_set_host_shapes(shapes)
    g = torch.Generator().manual_seed(zlib.crc32(c["id"].encode()))
    st, lsi, nv = level_geometry(shapes)
    st_d, lsi_d = st.to(DEV), lsi.to(DEV)
    orders = random_orders(b, nq, 7)
    order = orders[0] if c["order"] else None
    if kind == "plain":
        value, loc, attn = make_plain(b, shapes, M, D, P, nq, g, c["spread"])
        vb = value_buffer(value, c["strided"])
        loc_d, attn_d = (misaligned(t.to(DEV)) if c["misalign"] else t.to(DEV) for t in (loc, attn))

        def run(o):
            return forward_plain(pkg, vb, st_d, lsi_d, loc_d, attn_d, M, D, L, P, nv, o, sched)
        return run, order, orders, (value, loc, attn)
    value, ref, proj = make_fused(b, shapes, M, D, P, nq, g, 2 if kind == "fused2" else 4, c["spread"])
    vb = value_buffer(value, c["strided"])
    ref_d = ref.to(DEV)
    if c["misalign"]:  # a row stride of 3n + 1 floats: not a multiple of 4
        proj_d = torch.empty(b, nq, proj.shape[-1] + 1, device=DEV)[..., :proj.shape[-1]]
        proj_d.copy_(proj)
    else:
        proj_d = proj.to(DEV)

    def run(o):
        return pkg.cabi.msda_fused_forward(vb[0], vb[1], vb[2], vb[3], st_d, lsi_d, ref_d, proj_d, M, D, L, P, nv,
                                           o, sched, want_loc_attn=True)
    return run, order, orders, (value, ref, proj)


@pytest.mark.gpu
@pytest.mark.parametrize("c", FWD, ids=[c["id"] for c in FWD])
def test_forward_path(pkg, c):
    """One forward case: the output is within C_FWD of msda_ref (a fused run is checked in two steps: loc_out /
    attn_out against fused_ref, then the output against msda_ref at the kernel's own loc / attn); a repeated call and
    another query order give the same bits.  test_dispatch_launches_predicted_kernels checks which kernel it runs."""
    b, shapes, M, P, nq, kind = c["b"], c["shapes"], c["M"], c["P"], c["nq"], c["kind"]
    L = len(shapes)
    run, order, orders, host = setup_forward(pkg, c)
    family = predict_case(c)[0]
    res = run(order)
    out = res if kind == "plain" else res[0]
    if kind == "plain":
        value, loc, attn = host
    else:
        value, ref, proj = host
        _, loc_o, attn_o = (t.cpu() for t in res)
        want_loc, want_attn, shifted = fused_ref(ref, proj, shapes, M, L, P)
        fin = torch.isfinite(want_loc)
        assert torch.equal(torch.isfinite(loc_o), fin)
        nf = ~fin
        assert ((loc_o[nf] == want_loc[nf].float()) | (loc_o[nf].isnan() & want_loc[nf].isnan())).all()
        if kind == "fused2":
            hw = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
            term = proj[..., :2 * M * L * P].double().reshape(loc_o.shape).abs() / hw[None, None, None, :, None, :]
        else:
            term = (proj[..., :2 * M * L * P].double().reshape(loc_o.shape) / P).abs() * \
                ref[:, :, None, :, None, 2:].double() * 0.5
        sl = ref[:, :, None, :, None, :2].double().abs() + term
        r = within(torch.where(fin, loc_o, 0.0), torch.where(fin, want_loc, 0.0), torch.where(fin, sl, 0.0), C_LOC)
        assert r <= 1, r
        # __expf: at most 2 + 1.2 |x| ulp; the sum of NP terms and a reciprocal add NP + 2
        ax = shifted.abs().amax((-1, -2), keepdim=True)
        sa = (4 + 1.2 * ax + L * P) * want_attn
        r = within(attn_o, want_attn, sa, C_ATTN)
        assert r <= 1, r
        loc, attn = loc_o, attn_o
    want = msda_ref(value, shapes, loc, attn)
    r = within(out, want, forward_scale(value, shapes, loc, attn), C_FWD)
    assert r <= 1, (family, r)

    again = run(order)
    assert torch.equal(again if kind == "plain" else again[0], out)
    other = orders[1] if c["order"] else orders[0]
    if predict_case({**c, "order": True})[0] == family:
        moved = run(other)
        assert torch.equal(moved if kind == "plain" else moved[0], out)


@pytest.mark.gpu
def test_forward_byte_offsets_past_2_31(pkg):
    """A level whose token rows lie more than 2^31 bytes past the level start (368 640 tokens at a 6144-byte token
    stride, 2.3 GB): the 32-bit token index times the 32-bit byte stride of the gathers must widen to 64 bits."""
    shapes = [(640, 576), (16, 16), (8, 8), (4, 4)]
    st, lsi, nv = level_geometry(shapes)
    M, D, P, nq = 2, 32, 4, 200
    ts = 1536  # floats: 6144 bytes per token
    g = torch.Generator(device=DEV).manual_seed(0)
    buf = torch.empty(1, nv, ts, device=DEV)
    buf.normal_(generator=g)
    value = buf[:, :, 512:512 + M * D].reshape(1, nv, M, D)
    gl = torch.Generator().manual_seed(1)
    loc = torch.rand(1, nq, M, 4, P, 2, generator=gl)
    loc[:, : nq // 2, :, 0, :, 1] = 0.95 + 0.05 * loc[:, : nq // 2, :, 0, :, 1]  # rows past 349 526: beyond 2^31 bytes
    attn = torch.randn(1, nq, M, 4, P, generator=gl)
    loc_d, attn_d = loc.to(DEV), attn.to(DEV)
    pkg.cabi.msda_set_host_shapes(shapes)
    order = torch.randperm(nq, generator=gl).to(torch.int32)[None].to(DEV)
    want = msda_ref(value.double(), shapes, loc_d, attn_d).cpu()
    scale = msda_ref(value.double().abs(), shapes, loc_d, attn_d.abs()).cpu()
    st_d, lsi_d = st.to(DEV), lsi.to(DEV)
    vb = (buf, nv * ts, ts, 512)
    for sched, opts in ((0, {}), (1, {}), (1, {"msda_warp_per_item": 2}), (1, {"msda_tma": 1}),
                        (1, {"msda_smem_broadcast": 0})):
        for k, v in {**DEFAULTS, **opts}.items():
            pkg.cabi.set_option(k, v)
        out = forward_plain(pkg, vb, st_d, lsi_d, loc_d, attn_d, M, D, 4, P, nv, order, sched)
        assert within(out, want, scale, C_FWD) <= 1, (sched, opts)
    del buf, value
    torch.cuda.empty_cache()


# ---- backward ----------------------------------------------------------------------------------------------------------
def bcase(id, b, shapes, M, D, P, nq, gscale=1.0, collide=False):
    return dict(id=id, b=b, shapes=shapes, M=M, D=D, P=P, nq=nq, gscale=gscale, collide=collide)


BWD = [
    bcase("D4_L1_P1", 2, [(8, 16)], 3, 4, 1, 63),
    bcase("D8_L3_P2", 3, [(16, 8), (1, 1), (8, 1)], 1, 8, 2, 65),
    bcase("D16_L8_P8", 1, [(16, 16), (8, 8), (1, 8), (4, 4), (8, 1), (2, 2), (1, 1), (2, 4)], 3, 16, 8, 65),
    bcase("D32_L4_P4", 2, PROD, 8, 32, 4, 777),
    bcase("D64_L4_P4", 1, [(8, 16), (1, 1), (16, 1), (4, 4)], 3, 64, 4, 129),
    bcase("D128_L3_P2", 2, [(16, 32), (8, 16), (4, 8)], 1, 128, 2, 65),
    bcase("D32_tiny_grads", 2, PROD, 3, 32, 4, 129, gscale=1e-30),
    bcase("D32_huge_grads", 2, PROD, 3, 32, 4, 129, gscale=1e30),
    bcase("D128_tiny_grads", 1, [(16, 32), (8, 16), (4, 8)], 1, 128, 2, 65, gscale=1e-30),
    bcase("D4_huge_grads", 1, [(8, 16)], 2, 4, 8, 65, gscale=1e30),
    bcase("D32_collide", 1, [(4, 8)], 1, 32, 4, 4096, collide=True),
    bcase("D4_collide", 1, [(4, 8)], 2, 4, 4, 4096, collide=True),
]


def det_quantum(gout, attn, nq, P):
    """2^-s of the deterministic accumulation (msda_backward.cu: msda_det_scale_kernel): one unit of its int64 sums."""
    mg, ma = float(gout.abs().max()), float(attn.abs().max())
    if mg == 0 or ma == 0:
        return 0.0
    ec = max(0, math.ceil(math.log2(nq * P)))
    return 2.0 ** (math.frexp(mg)[1] + math.frexp(ma)[1] + ec - 62)


def setup_backward(c):
    """-> (value, loc, attn, grad_out) on the host, the device arguments of msda_backward, the generator."""
    b, shapes, M, D, P, nq = c["b"], c["shapes"], c["M"], c["D"], c["P"], c["nq"]
    g = torch.Generator().manual_seed(zlib.crc32(c["id"].encode()))
    value, loc, attn = make_plain(b, shapes, M, D, P, nq, g)
    if c["collide"]:  # every sample inside the 2x2 neighbourhood of tokens (1..2, 3..4) of the 4x8 map
        H, W = shapes[0]
        loc[..., 0] = (3.5 + torch.rand(loc[..., 0].shape, generator=g)) / W
        loc[..., 1] = (1.5 + torch.rand(loc[..., 1].shape, generator=g)) / H
        loc[:, ::7, ..., 0] = 3.5 / W  # exact pixel centres
    gout = torch.randn(b, nq, M * D, generator=g) * c["gscale"]
    st, lsi, _ = level_geometry(shapes)
    return value, loc, attn, gout, [t.to(DEV) for t in (value, st, lsi, loc, attn, gout)], g


@pytest.mark.gpu
@pytest.mark.parametrize("c", BWD, ids=[c["id"] for c in BWD])
def test_backward_path(pkg, c):
    """Atomic and deterministic backward: all three gradients within their bounds of msda_ref's autograd; deterministic
    grad_loc / grad_attn bit-identical to the atomic ones; deterministic grad_value bit-identical across repeats and
    query permutations.  test_dispatch_launches_predicted_kernels checks which kernels run."""
    value, loc, attn, gout, args, g = setup_backward(c)
    shapes, P, nq = c["shapes"], c["P"], c["nq"]
    gv, gl, ga = pkg.cabi.msda_backward(*args)
    dv, dl, da = pkg.cabi.msda_backward_deterministic(*args)
    rv, rl, ra = reference_grads(value, shapes, loc, attn, gout)
    sv, sa, sl = backward_scales(value, shapes, loc, attn, gout)
    # an element of grad_value receives at most nq * P additions: each float atomic can flush up to FLT_MIN, each
    # fixed-point one rounds by half a quantum
    for tag, got, want, s, cc, t in (("gv", gv, rv, sv, C_GV, TINY + nq * P * FLT_MIN), ("ga", ga, ra, sa, C_GA, TINY),
                                      ("gl", gl, rl, sl, C_GL, TINY),
                                      ("dv", dv, rv, sv, C_GV, TINY + nq * P * det_quantum(gout, attn, nq, P))):
        r = within(got, want, s, cc, t)
        assert r <= 1, (tag, r)
    assert torch.equal(dl, gl) and torch.equal(da, ga)
    dv2, dl2, da2 = pkg.cabi.msda_backward_deterministic(*args)
    assert torch.equal(dv2, dv) and torch.equal(dl2, dl) and torch.equal(da2, da)
    perm = torch.randperm(nq, generator=g)
    pargs = [args[0], args[1], args[2], args[3][:, perm].contiguous(), args[4][:, perm].contiguous(),
             args[5][:, perm].contiguous()]
    pv, pl, pa = pkg.cabi.msda_backward_deterministic(*pargs)
    assert torch.equal(pv, dv) and torch.equal(pl, dl[:, perm]) and torch.equal(pa, da[:, perm])


def dispatch_sequence(pkg):
    """Launch one case of every distinct dispatch key of the forward table, then every backward case (atomic, then
    deterministic), in one profiler session -> (predicted (family, kernel) list, names of the MSDA kernels that ran, in
    launch order, the tail as long as the prediction)."""
    from torch.profiler import ProfilerActivity, profile
    firsts = {}
    for c in FWD:
        firsts.setdefault(dispatch_key(c), c)
    want = [predict_case(c) for c in firsts.values()]
    want += [(f"B{c['D']}{s}", f"msda_bwd_kernel<{c['D']}, {d}>") for c in BWD for s, d in (("", "false"), ("det", "true"))]
    warm = setup_forward(pkg, FWD[0])
    for _ in range(3):  # the profiler may drop launches made right after it starts: a lossy session is repeated
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.05)
            for _ in range(3):
                warm[0](warm[1])
            torch.cuda.synchronize()
            for c in firsts.values():
                run, order, _, _ = setup_forward(pkg, c)
                run(order)
                torch.cuda.synchronize()
            for k, v in DEFAULTS.items():
                pkg.cabi.set_option(k, v)
            for c in BWD:
                args = setup_backward(c)[4]
                pkg.cabi.msda_backward(*args)
                pkg.cabi.msda_backward_deterministic(*args)
                torch.cuda.synchronize()
        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
              and ("msda_fwd" in e.name or "msda_bwd" in e.name)]
        if len(ev) >= len(want) + 2:  # at most the first warm-up launch missing
            break
    return want, [e.name for e in sorted(ev, key=lambda e: e.time_range.start)][-len(want):]


@pytest.mark.gpu
def test_dispatch_launches_predicted_kernels():
    """The sequence of MSDA kernels on the device is the predicted one, and it covers F1-F6 and both backward flavours
    at every head dim.  The session runs in a child process: once the profiler has run in a process, later GPU work there
    (other test files) can stop it from recording kernels, which would break the profiler checks of later tests.  One
    session, one case per dispatch key: the dispatch depends on nothing but the key, so this confirms every case."""
    code = ("import json, sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_msda_paths as t; "
            "import salience_detr_b200 as p; print(json.dumps(t.dispatch_sequence(p)))")
    tests = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-s", "-c", code, os.path.dirname(tests), tests], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    want, got = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(got) == len(want)
    for (family, name), g in zip(want, got):
        assert name in g, (family, name, g)
    families = {f for f, _ in want}
    assert families == {"F1", "F2", "F3", "F4", "F5", "F6"} | {f"B{d}{s}" for d in (4, 8, 16, 32, 64, 128) for s in ("", "det")}
