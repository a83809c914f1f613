"""The encoder layer's fused GEMM epilogues against the unfused pairs they replace, bit for bit:
* sdetr_gemm_f16x3_rowmax = sdetr_gemm_f16x3_pre (class scores) + sdetr_class_max_times_fg;
* sdetr_gemm_f16x3_add_layernorm = sdetr_gemm_f16x3_pre (output projection) + sdetr_add_layernorm(q, ., out=q) (norm1).
Row counts around the 64 / 128-row boundaries, one row and the six encoder layers of the bench workload; non-finite
logits and activations, rows of mean 1e4 and std 1e-2, capped persistent grids; float64 bounds as a second line."""
import pytest
import torch
import torch.nn.functional as F

DEV = "cuda:0"
LAYER_ROWS = (22726, 18180, 13634, 13634, 9090, 4544)  # bs = 2 at the bench workload
ROWS = (1, 63, 64, 65, 127, 128, 129, 191, 255, 257, 2305) + LAYER_ROWS


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


def bits(t):
    return t.contiguous().view(torch.int32)


def split(pkg, w):
    return pkg.cabi.split_f16_pair(w)


def rowmax_pair(pkg, x, wp, b, fg):
    old = pkg.cabi.class_max_times_fg(pkg.cabi.gemm_f16x3_pre(x, *wp, b), fg)
    new = pkg.cabi.gemm_f16x3_rowmax(x, *wp, b, fg)
    return old, new


def ln_pair(pkg, q, x, wp, b, gam, bet, eps=1e-5):
    old = q.clone()
    pkg.cabi.add_layernorm(old, pkg.cabi.gemm_f16x3_pre(x, *wp, b), gam, bet, eps, out=old)
    new = pkg.cabi.gemm_f16x3_add_layernorm_(q.clone(), x, *wp, b, gam, bet, eps)
    return old, new


def ln64(q, x, w, b, gam, bet, eps=1e-5):
    v = q.double() + F.linear(x.double(), w.double(), b.double())
    mean, var = v.mean(-1, keepdim=True), v.var(-1, unbiased=False, keepdim=True)
    y = (v - mean) / torch.sqrt(var + eps) * gam.double() + bet.double()
    # fp32 rounding of v (|v| 2^-24 each) and of the product, amplified by 1 / std
    bound = 64 * 2.0 ** -24 * (v.abs().amax(-1, keepdim=True) + 1) / torch.sqrt(var + eps) * gam.double().abs() + 1e-6
    return y, bound


def layer_inputs(M, g, N=91):
    x = torch.randn(M, 256, generator=g).to(DEV)
    w = (torch.randn(N, 256, generator=g) / 16).to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    return x, w, b


@pytest.mark.gpu
@pytest.mark.parametrize("M", ROWS)
def test_rowmax_bits(pkg, M):
    g = torch.Generator().manual_seed(M)
    for N in ((91, 1, 64, 128) if M <= 2305 else (91,)):
        x, w, b = layer_inputs(M, g, N)
        fg = torch.rand(M, generator=g).to(DEV)
        old, new = rowmax_pair(pkg, x, split(pkg, w), b, fg)
        assert torch.equal(bits(old), bits(new)), (M, N)
        ref = (F.linear(x.double(), w.double(), b.double()).amax(-1) * fg.double())
        S = F.linear(x.double().abs(), w.double().abs(), b.double().abs()).amax(-1) * fg.double()
        assert ((new.double() - ref).abs() <= 64 * 2.0 ** -24 * S + 1e-6).all(), (M, N)
    old, new = rowmax_pair(pkg, x, split(pkg, w), None, fg)  # no bias
    assert torch.equal(bits(old), bits(new)), M


@pytest.mark.gpu
def test_rowmax_nonfinite_and_signed_zero(pkg):
    g = torch.Generator().manual_seed(5)
    M = 3000
    x, w, b = layer_inputs(M, g)
    fg = torch.rand(M, generator=g).to(DEV)
    fg[7], fg[8] = -0.0, 0.0
    x[11, 5] = float("nan")     # a NaN activation poisons its own row only
    x[12, 9] = float("inf")      # inf -> NaN in the fp16 split
    x[13] = 0.0                  # logits = bias
    wp = split(pkg, w)
    clean_old, _ = rowmax_pair(pkg, torch.where(torch.isfinite(x), x, torch.zeros_like(x)), wp, b, fg)
    old, new = rowmax_pair(pkg, x, wp, b, fg)
    assert torch.equal(bits(old), bits(new))
    assert new[11].isnan() and new[12].isnan()
    keep = torch.ones(M, dtype=torch.bool, device=DEV)
    keep[11:13] = False
    assert torch.equal(bits(new[keep]), bits(clean_old[keep]))
    for special in (float("nan"), float("inf"), -float("inf"), -0.0, 0.0):
        for col in (0, 45, 90):
            bs = b.clone()
            bs[col] = special
            bs[(col + 1) % 91] = -0.0
            old, new = rowmax_pair(pkg, x, wp, bs, fg)
            assert torch.equal(bits(old), bits(new)), (special, col)
    # every logit a signed zero: zero weights, a bias of zeros of both signs
    bz = torch.zeros(91, device=DEV)
    bz[::2] = -0.0
    old, new = rowmax_pair(pkg, x, split(pkg, torch.zeros_like(w)), bz, fg)
    assert torch.equal(bits(old), bits(new))


@pytest.mark.gpu
@pytest.mark.parametrize("M", ROWS)
def test_add_layernorm_bits(pkg, M):
    g = torch.Generator().manual_seed(100 + M)
    x, w, b = layer_inputs(M, g, 256)
    q = torch.randn(M, 256, generator=g).to(DEV)
    gam, bet = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV), (0.1 * torch.randn(256, generator=g)).to(DEV)
    old, new = ln_pair(pkg, q, x, split(pkg, w), b, gam, bet)
    assert torch.equal(bits(old), bits(new)), M
    ref, bound = ln64(q, x, w, b, gam, bet)
    assert ((new.double() - ref).abs() <= bound).all(), M
    old, new = ln_pair(pkg, q, x, split(pkg, w), None, gam, bet)  # no bias
    assert torch.equal(bits(old), bits(new)), M


@pytest.mark.gpu
def test_add_layernorm_nonfinite_rows_and_large_mean(pkg):
    g = torch.Generator().manual_seed(9)
    M = 2500
    x, w, b = layer_inputs(M, g, 256)
    q = torch.randn(M, 256, generator=g).to(DEV)
    q[100:200] = 1e4 + 1e-2 * torch.randn(100, 256, generator=g).to(DEV)  # mean 1e4, std 1e-2
    x[100:200] *= 1e-4
    gam, bet = (1 + 0.1 * torch.randn(256, generator=g)).to(DEV), (0.1 * torch.randn(256, generator=g)).to(DEV)
    wp = split(pkg, w)
    clean, _ = ln_pair(pkg, q, x, wp, b, gam, bet)
    ref, bound = ln64(q, x, w, b, gam, bet)
    assert ((clean.double() - ref).abs() <= bound).all()
    x[7, 3] = float("nan")    # NaN activation row
    q[9, 200] = float("inf")  # inf residual
    q[10, 0] = -0.0
    old, new = ln_pair(pkg, q, x, wp, b, gam, bet)
    assert torch.equal(bits(old), bits(new))
    assert new[7].isnan().all() and new[9].isnan().all()
    keep = torch.ones(M, dtype=torch.bool, device=DEV)
    keep[7] = keep[9] = False
    keep[10] = False
    assert torch.equal(bits(new[keep]), bits(clean[keep]))


@pytest.mark.gpu
def test_capped_persistent_grids(pkg):
    g = torch.Generator().manual_seed(13)
    M = 4544  # 36 panels of 128 rows
    x, w, b = layer_inputs(M, g)
    fg = torch.rand(M, generator=g).to(DEV)
    xl, wl, bl = layer_inputs(M, g, 256)
    q = torch.randn(M, 256, generator=g).to(DEV)
    gam, bet = torch.rand(256, generator=g).to(DEV), torch.randn(256, generator=g).to(DEV)
    wp, wlp = split(pkg, w), split(pkg, wl)
    want_max = pkg.cabi.gemm_f16x3_rowmax(x, *wp, b, fg)
    want_ln = pkg.cabi.gemm_f16x3_add_layernorm_(q.clone(), xl, *wlp, bl, gam, bet)
    try:
        for cap in (1, 2, 5, 35):
            pkg.cabi.lib().sdetr_set_persistent_ctas(cap)
            assert torch.equal(bits(pkg.cabi.gemm_f16x3_rowmax(x, *wp, b, fg)), bits(want_max)), cap
            got = pkg.cabi.gemm_f16x3_add_layernorm_(q.clone(), xl, *wlp, bl, gam, bet)
            assert torch.equal(bits(got), bits(want_ln)), cap
    finally:
        pkg.cabi.lib().sdetr_set_persistent_ctas(0)


@pytest.mark.gpu
def test_entry_points_reject_bad_shapes(pkg):
    x = torch.randn(300, 256, device=DEV)
    w = torch.randn(129, 256, device=DEV)
    with pytest.raises(RuntimeError):
        pkg.cabi.gemm_f16x3_rowmax(x, *split(pkg, w), None, torch.ones(300, device=DEV))  # N > 128
    with pytest.raises(RuntimeError):
        pkg.cabi.gemm_f16x3_add_layernorm_(torch.randn(300, 128, device=DEV), x, *split(pkg, torch.randn(256, 256, device=DEV)),
                                           None, torch.ones(256, device=DEV), torch.zeros(256, device=DEV))
