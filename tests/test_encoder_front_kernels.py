"""The encoder's front end and the salience-score head on every launch path, against float64 and bit-exact torch.

Front end: `flatten_routes` restates the host routing of flatten_tokens_impl (csrc/tokens.cu): a level goes to the
vectorised kernel (16-token tiles, grid.y in steps of 256 channels) when its token count is a multiple of 4, C % 4 == 0
and its maps are 16-byte aligned; every other level goes to the shared-memory tile kernel (32-token tiles, grid.y in steps
of 32 channels).  A case table reaches both routes, a tile level by size and one by pointer alignment, 1 and kMaxLevels
levels; both entry points, token_lpos_keep and token_map_transpose are compared bit for bit with torch.

gelu_colmean: `colmean_grid` restates the chunk counts (chunks1 capped at 4 SMs / batch, chunks2 at SMs / batch) from the
device's SM count; the workspace bound is checked against it.  mask_predictor_level (csrc/predictor_small.cu): the fused
small-level route against MaskPredictor in float64, and the encoder's score loop on both sides of the 4096-row route
boundary.  mask_plan / sine_pos_tokens (csrc/plan.cu) and salience_targets against the torch restatements.

Bounds are |got - ref| <= c * 2^-24 * S element-wise, S built from the same float64 computation on absolute values.
SDETR_FRONT_OBSERVE=1 prints the largest c every bound needed (calibration)."""
import math
import os
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

DEV = "cuda:0"
U = 2.0 ** -24  # unit round-off of float32
H100_SMS = 132

# Bound constants c of |got - ref| <= c * 2^-24 * S.  Each is about four times the largest c observed over every case of
# this file on an H100 80GB HBM3 at 700 W (noted beside it).
C_GELU = 4.0    # gelu_colmean's local half: S = |x| + |GELU(x)| (observed 0.975)
C_MEAN = 1.5    # gelu_colmean's mean columns: S = (1 + n) max_rows(|x| + |GELU(x)|) (observed 0.377)
C_PRED = 2e-4   # mask_predictor_level: S composes every stage's scale, which overstates the error by about 10^4
                #   (observed 5.29e-5)
C_LOOP = 3e-4   # the encoder's score loop, fused and forward_fast routes, S as for C_PRED (observed 8.01e-5)
C_SINE = 3.5    # sine_pos_tokens: S = 1 + |e / dim_t| (observed 0.848)
C_TGT = 5.0     # salience_targets: S = 1 (observed 1.15)

OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    if os.environ.get("SDETR_FRONT_OBSERVE"):
        print("\nOBSERVED", {k: float(f"{v:.3g}") for k, v in sorted(OBSERVED.items())})


def check_bound(name, got, ref, S, c):
    """|got - ref| <= c u S element-wise (NaN anywhere fails); records the c the case needed."""
    err = (got.detach().double().cpu() - ref).abs()
    need = (err / (U * S).clamp_min(1e-300)).masked_fill((S == 0) & (err == 0), 0)
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(need.max()) if need.numel() else 0.0)
    bad = ~(err <= c * U * S)
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} of {bad.numel()} outside c={c} (needs {float(need.max()):.3g})"


def same_bits(got, want):
    """Bit-identical float32 tensors, a NaN only where the other has one."""
    got, want = got.detach().cpu(), want.detach().cpu()
    if got.shape != want.shape or got.dtype != want.dtype:
        return False
    nan = torch.isnan(want)
    if not torch.equal(torch.isnan(got), nan):
        return False
    return torch.equal(got.masked_fill(nan, 0).view(torch.int32), want.masked_fill(nan, 0).view(torch.int32))


def flatten_levels(xs):
    """(b, [C], H, W) per level -> (b, Nv, [C]) tokens (base_transformer.py:21-26)."""
    y = torch.cat([e.flatten(-2) for e in xs], -1)
    return y.transpose(1, 2).contiguous() if y.ndim == 3 else y


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ==== 1. flatten and the layout hand-off ================================================================================
MAX_LEVELS = 8  # kMaxLevels


def flatten_routes(sizes, ptrs, C, vectorised=True, shared=()):
    """flatten_tokens_impl's routing: per level "vec" or "tile", and the two grids.  ptrs: per level the addresses of its
    maps (feature, and position unless the position comes in token layout); shared: the addresses every level uses (the
    three outputs, level_embeds, position tokens)."""
    vec_ok = vectorised and C % 4 == 0 and all(p % 16 == 0 for p in shared)
    routes = ["vec" if vec_ok and hw % 4 == 0 and all(p % 16 == 0 for p in ps) else "tile" for hw, ps in zip(sizes, ptrs)]
    vt = sum(-(-hw // 16) for hw, r in zip(sizes, routes) if r == "vec")
    rt = sum(-(-hw // 32) for hw, r in zip(sizes, routes) if r == "tile")
    grids = {"vec": (vt, -(-C // 256)) if vt else None, "tile": (rt, -(-C // 32)) if rt else None}
    return routes, grids


# (b, C, level shapes, levels whose maps sit 4 bytes past a 16-byte boundary)
FLATTEN_CASES = [
    (3, 4, [(4, 5), (3, 3)], ()),                                                       # vec + tile by size, C = 4
    (1, 36, [(8, 8), (5, 7), (4, 4), (3, 3), (2, 2), (1, 4), (1, 1), (2, 6)], (2, 7)),  # 8 levels, tile by alignment
    (3, 256, [(12, 20)], ()),                                                           # 1 level, vectorised
    (1, 256, [(13, 21)], ()),                                                           # 1 level, tile by size
    (1, 260, [(16, 16), (7, 11), (1, 4)], (0,)),                                        # a partial 256-channel block
    (3, 1024, [(6, 8), (3, 5), (2, 2)], (2,)),
    (1, 1024, [(1, 1), (2, 2), (3, 4), (5, 5), (4, 6), (1, 9), (7, 1), (8, 4)], (4,)),
]


def _case_routes(b, C, shapes, mis, vectorised=True):
    """Routes of a table row with its maps at 16-byte-aligned addresses, the misaligned levels at 4 bytes past one."""
    sizes = [h * w for h, w in shapes]
    ptrs = [((4 if l in mis else 0), (4 if l in mis else 0)) for l in range(len(shapes))]
    return flatten_routes(sizes, ptrs, C, vectorised)[0]


def test_flatten_case_table_reaches_every_route():
    routes = [(_case_routes(b, C, s, mis), b, C, s, mis) for b, C, s, mis in FLATTEN_CASES]
    kinds = set()
    for r, b, C, shapes, mis in routes:
        for l, ((h, w), k) in enumerate(zip(shapes, r)):
            kinds.add(k if k == "vec" else ("tile_align" if (h * w) % 4 == 0 else "tile_size"))
            assert (k == "tile") == ((h * w) % 4 != 0 or l in mis)
    assert kinds == {"vec", "tile_size", "tile_align"}
    assert any({"vec", "tile"} <= set(r) for r, *_ in routes)  # both kernels in one call
    assert {len(s) for *_, s, _ in routes} >= {1, MAX_LEVELS}
    assert {C for _, _, C, _, _ in routes} == {4, 36, 256, 260, 1024} and {b for _, b, *_ in routes} == {1, 3}
    assert any(-(-C // 256) > 1 for _, _, C, _, _ in routes)  # vec grid.y > 1
    assert all(set(_case_routes(b, C, s, mis, vectorised=False)) == {"tile"} for b, C, s, mis in FLATTEN_CASES)


def _maps(vals, misaligned):
    """A device copy of vals, at an address 4 bytes past a 16-byte boundary when misaligned."""
    if not misaligned:
        return vals.to(DEV)
    buf = torch.empty(vals.numel() + 4, device=DEV)
    out = buf[1:1 + vals.numel()].view(vals.shape)
    out.copy_(vals)
    assert out.data_ptr() % 16 == 4 and out.is_contiguous()
    return out


def _flatten_inputs(b, C, shapes, mis, seed):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
    pos = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
    emb = torch.randn(len(shapes), C, generator=g)
    nv = sum(h * w for h, w in shapes)
    keep = (torch.rand(b, nv, generator=g) > 0.3).float()
    keep[0, 0] = 0.5  # a keep weight that is not 0 or 1: the multiply is checked, not just a select
    fd = [_maps(f, l in mis) for l, f in enumerate(feats)]
    pd = [_maps(p, l in mis) for l, p in enumerate(pos)]
    return feats, pos, emb, keep, fd, pd


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FLATTEN_CASES)))
def test_flatten_both_entry_points_bit_exact(pkg, case):
    """flatten_tokens and flatten_tokens_pos against flatten_levels + level_embeds[l] + keep, bit for bit, with the
    vectorised kernel on and off; the launch count is the number of routes flatten_routes predicts; token_lpos_keep gives
    the same lpos and x bits."""
    b, C, shapes, mis = FLATTEN_CASES[case]
    feats, pos, emb, keep, fd, pd = _flatten_inputs(b, C, shapes, mis, 500 + case)
    want_f = flatten_levels(feats)
    want_p = flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, emb)])
    want_x = (want_f + want_p) * keep[..., None]
    pos_tok = flatten_levels(pos).to(DEV)
    sizes = [h * w for h, w in shapes]
    embd, keepd = emb.to(DEV), keep.to(DEV)
    lib = pkg.cabi.lib()
    for vec in (1, 0):
        lib.sdetr_flatten_set_vectorized(vec)
        try:
            for name, call, ptrs in (("maps", lambda: pkg.cabi.flatten_tokens(fd, pd, embd, keepd),
                                      [(f.data_ptr(), p.data_ptr()) for f, p in zip(fd, pd)]),
                                     ("tokens", lambda: pkg.cabi.flatten_tokens_pos(fd, pos_tok, embd, keepd),
                                      [(f.data_ptr(),) for f in fd])):
                routes, _ = flatten_routes(sizes, ptrs, C, bool(vec), shared=(embd.data_ptr(), pos_tok.data_ptr()))
                n0 = pkg.cabi.launch_count()
                f, p, x = call()
                assert pkg.cabi.launch_count() - n0 == len(set(routes)), (name, vec, routes)
                assert same_bits(f, want_f) and same_bits(p, want_p) and same_bits(x, want_x), (name, vec, routes)
        finally:
            lib.sdetr_flatten_set_vectorized(1)
    lpos, x = pkg.cabi.token_lpos_keep(want_f.to(DEV), pos_tok, embd, keepd, sizes)
    assert same_bits(lpos, want_p) and same_bits(x, want_x)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(FLATTEN_CASES)))
def test_token_map_transpose_both_directions(pkg, case):
    """tokens_to_maps equals torch's split / transpose / reshape, maps_to_tokens equals flatten(2) / transpose / cat (also
    from misaligned maps), and the round trip is the identity, bit for bit."""
    b, C, shapes, mis = FLATTEN_CASES[case]
    g = torch.Generator().manual_seed(600 + case)
    sizes = [h * w for h, w in shapes]
    tokens = torch.randn(b, sum(sizes), C, generator=g)
    maps = pkg.cabi.tokens_to_maps(tokens.to(DEV), shapes)
    want = [t.transpose(1, 2).reshape(b, C, h, w) for t, (h, w) in zip(tokens.split(sizes, 1), shapes)]
    assert all(same_bits(m, w) for m, w in zip(maps, want))
    assert same_bits(pkg.cabi.maps_to_tokens(maps), tokens)
    src = [torch.randn(b, C, h, w, generator=g) for h, w in shapes]
    got = pkg.cabi.maps_to_tokens([_maps(s, l in mis) for l, s in enumerate(src)])
    assert same_bits(got, flatten_levels(src))
    assert all(same_bits(m, s) for m, s in zip(pkg.cabi.tokens_to_maps(got, shapes), src))


# ==== 2. gelu_colmean ===================================================================================================
MEAN_THREADS = 256


def colmean_grid(b, n, sms):
    """sdetr_gelu_colmean's chunk counts: (chunks1 of the column-sum pass, chunks2 of the broadcast pass)."""
    return min(-(-n // 32), max(4 * sms // b, 1)), min(-(-n // 64), max(sms // b, 1))


# (b, n, C, half)
GELU_CASES = [
    (1, 1, 12, 4), (3, 1, 12, 0), (2, 37, 12, 8),
    (2, 1000, 96, 48), (1, 273, 96, 4), (3, 50, 96, 92), (2, 5, 96, 0),
    (2, 16800, 256, 128), (8, 16800, 256, 128), (1, 273, 256, 0), (4, 999, 256, 252), (3, 300, 256, 4),
    (1, 2000, 1020, 508), (2, 33, 1020, 1016), (1, 64, 1020, 4), (2, 77, 1020, 0),
    (1, 700, 1024, 512), (2, 1, 1024, 0), (600, 3, 1024, 4), (1, 129, 1024, 1020),
]


def assert_colmean_reach(sms):
    grids = [(c, colmean_grid(c[0], c[1], sms)) for c in GELU_CASES]
    assert any(g[0] == -(-c[1] // 32) and c[1] > 32 for c, g in grids)           # uncapped
    assert any(g[0] < -(-c[1] // 32) and g[0] > 1 for c, g in grids)             # capped by 4 SMs / batch
    assert any(c[0] > 4 * sms and g[0] == 1 for c, g in grids)                   # capped at one chunk
    assert (8, 16800, 256, 128) in [c for c, _ in grids] and any(c[1] == 1 for c, _ in grids)
    assert any(MEAN_THREADS % (c[2] // 4) for c, _ in grids)                     # idle threads in the sum pass
    assert any(MEAN_THREADS % ((c[2] - c[3]) // 4) for c, _ in grids)            # idle threads in the broadcast pass
    for C in (12, 96, 256, 1020, 1024):
        halves = {c[3] for c, _ in grids if c[2] == C}
        assert {0, 4, C - 4} <= halves and (C // 2 % 4 or C // 2 in halves), C


def test_gelu_colmean_case_table_reaches_every_regime():
    assert_colmean_reach(H100_SMS)
    assert colmean_grid(8, 16800, H100_SMS) == (66, 16) and colmean_grid(1, 273, H100_SMS) == (9, 5)


def gelu64(x):
    return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))


def colmean_ref(z, half):
    """float64 GELU with the columns [half, C) replaced by their per-image token mean, and the S of each element:
    |x| + |GELU(x)| on the local half; on the mean columns the GELU's own scale plus the n-term sum's, (1 + n) times the
    largest |x| + |GELU(x)| of the image's rows."""
    x = z.double()
    g = gelu64(x)
    S = x.abs() + g.abs()
    ref, Sr = g.clone(), S.clone()
    n = x.shape[1]
    ref[..., half:] = g[..., half:].mean(1, keepdim=True)
    Sr[..., half:] = (1 + n) * S[..., half:].amax(1, keepdim=True)
    return ref, Sr


@pytest.mark.gpu
def test_gelu_colmean_case_table_reaches_every_regime_on_device():
    assert_colmean_reach(_sms())


@pytest.mark.gpu
def test_gelu_colmean_workspace_covers_the_partials(pkg):
    """sdetr_gelu_colmean_workspace holds batch * chunks1 * (C - half) floats for every batch up to 4096 on this device."""
    lib, sms = pkg.cabi.lib(), _sms()
    for b in list(range(1, 1200)) + [4096]:
        for n in (1, 16800, 1 << 20):
            c1 = colmean_grid(b, n, sms)[0]
            for C, half in ((1024, 0), (256, 128), (12, 8)):
                assert lib.sdetr_gelu_colmean_workspace(b, n, C, half) >= 4 * b * c1 * (C - half), (b, n, C, half)


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(GELU_CASES)))
def test_gelu_colmean_vs_float64(pkg, case):
    """The local half within C_GELU of float64 GELU, the mean columns within C_MEAN (1 + n) u max(|x| + |GELU|) of the
    float64 mean; one mean column at 1e4 + N(0, 1); a repeat gives the same bits.  One mean column of integers in
    [8, 900] is exact: GELU is the identity there in float32 and every partial sum is an integer below 2^24, so the mean
    is the float32 quotient sum / n bit for bit, and a row left out of (or added twice to) the sum shows."""
    b, n, C, half = GELU_CASES[case]
    g = torch.Generator().manual_seed(zlib.crc32(f"gelu{b},{n},{C},{half}".encode()))
    z = torch.randn(b, n, C, generator=g) * 2
    z[..., C - 4] = 1e4 + torch.randn(b, n, generator=g)
    ints = torch.randint(8, 901, (b, n), generator=g)
    z[..., C - 3] = ints.float()
    assert int(ints.sum(1).max()) < 2 ** 24
    ref, S = colmean_ref(z, half)
    got = pkg.cabi.gelu_colmean_(z.to(DEV), half)
    exact = ints.sum(1).float() / torch.tensor(float(n))
    assert same_bits(got[:, 0, C - 3], exact)
    check_bound("gelu_local", got[..., :half], ref[..., :half], S[..., :half], C_GELU)
    check_bound("gelu_mean", got[..., half:], ref[..., half:], S[..., half:], C_MEAN)
    assert same_bits(got[..., half:], got[:, :1, half:].expand(-1, n, -1).contiguous())  # one mean per (image, column)
    assert torch.equal(pkg.cabi.gelu_colmean_(z.to(DEV), half), got)


@pytest.mark.gpu
def test_gelu_colmean_nan_stays_in_its_image(pkg):
    """A NaN in a mean column makes that column of its own image NaN; a NaN in a local column stays in its element; every
    other value is bit-identical to the clean run (both grid regimes)."""
    g = torch.Generator().manual_seed(8)
    for b, n, C, half in ((3, 300, 256, 128), (8, 16800, 256, 128), (2, 40, 96, 4)):
        z = torch.randn(b, n, C, generator=g)
        clean = pkg.cabi.gelu_colmean_(z.to(DEV), half).cpu()
        bad = z.clone()
        bad[1, n // 2, half + 3] = float("nan")
        bad[1, n - 1, half // 2] = float("nan") if half else bad[1, n - 1, half // 2]
        got = pkg.cabi.gelu_colmean_(bad.to(DEV), half).cpu()
        nan = torch.zeros(b, n, C, dtype=torch.bool)
        nan[1, :, half + 3] = True
        if half:
            nan[1, n - 1, half // 2] = True
        assert torch.equal(torch.isnan(got), nan), (b, n, C, half)
        assert same_bits(got[~nan], clean[~nan])


# ==== 3. mask_predictor_level ===========================================================================================
def _predictor(seed):
    from salience_detr_b200.salience_transformer import MaskPredictor
    g = torch.Generator().manual_seed(seed)
    mp = MaskPredictor(256, 256)
    with torch.no_grad():
        for p in mp.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.08 if p.dim() > 1 else 0.2))
        mp.layer1[0].weight.add_(1.0)
    return mp


def modulate_ref(mem, coarse, alpha, H, W, Hc, Wc, S_coarse=None):
    """float64 mem + mem * up * alpha, up the align_corners=True bilinear resize at ATen's float32 source coordinates, and
    the S of its bound (in units of u, absolute); S_coarse: the error scale the coarse scores carry."""
    def axis(n_out, n_in):
        s = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
        f = (s * np.arange(n_out, dtype=np.float32)).astype(np.float32)
        i0 = f.astype(np.int64)
        i1 = np.minimum(i0 + 1, n_in - 1)
        lam = torch.from_numpy((f - i0.astype(np.float32)).astype(np.float64))
        return torch.from_numpy(i0), torch.from_numpy(i1), lam

    y0, y1, ly = axis(H, Hc)
    x0, x1, lx = axis(W, Wc)
    b = mem.shape[0]

    def up_of(cs):
        cs = cs.double().reshape(b, Hc, Wc)
        terms = [((1 - ly)[:, None] * (1 - lx)[None], cs[:, y0][:, :, x0]), ((1 - ly)[:, None] * lx[None], cs[:, y0][:, :, x1]),
                 (ly[:, None] * (1 - lx)[None], cs[:, y1][:, :, x0]), (ly[:, None] * lx[None], cs[:, y1][:, :, x1])]
        return sum(w * v for w, v in terms).view(b, H * W, 1), sum(w * v.abs() for w, v in terms).view(b, H * W, 1)

    up, up_abs = up_of(coarse)
    m = mem.double()
    ref = m + m * up * alpha
    S = m.abs() + (m * alpha).abs() * (up.abs() + up_abs)
    if S_coarse is not None:
        S = S + (m * alpha).abs() * up_of(S_coarse)[1]
    return ref, S


GELU_LIP = 1.13  # max |GELU'|


def predictor_ref(mp64, m, E):
    """float64 MaskPredictor of m (b, HW, 256) and the S of its bound: each stage adds its own rounding scale (|W| |x| + |b|
    of a linear layer, |x| of a GELU, the summation depth of the token mean: 8 rows of a tile, then half the tiles) to the
    propagated scale of its input (through |W|, through GELU's Lipschitz constant).  E: the error scale m carries in."""
    ln, fc1 = mp64.layer1[0], mp64.layer1[1]
    fc2a, fc2b, fc2c = mp64.layer2[0], mp64.layer2[2], mp64.layer2[4]
    m = m.double()
    mu = m.mean(-1, keepdim=True)
    d = m - mu
    rstd = 1 / torch.sqrt((d * d).mean(-1, keepdim=True) + ln.eps)
    zhat = d * rstd
    A = E + m.abs()
    Ab = A.mean(-1, keepdim=True)
    gam, bet = ln.weight.detach(), ln.bias.detach()
    x = zhat * gam + bet
    S = gam.abs() * rstd * (A + Ab) + (gam * zhat).abs() * (1 + rstd * rstd * (d.abs() * (A + Ab)).mean(-1, keepdim=True)) + bet.abs()

    def linear(x, S, lin):
        w, bias = lin.weight.detach(), lin.bias.detach()
        return x @ w.t() + bias, (x.abs() + S) @ w.abs().t() + bias.abs()

    def gelu(y, S):
        return gelu64(y), GELU_LIP * S + y.abs()

    y, S = gelu(*linear(x, S, fc1))
    HW = m.shape[1]
    depth = 8 + (-(-HW // 8)) // 2 + 2
    y = torch.cat([y[..., :128], y[..., 128:].mean(1, keepdim=True).expand(-1, HW, -1)], -1)
    S = torch.cat([S[..., :128], (S[..., 128:].mean(1, keepdim=True) + depth * y[..., 128:].abs().mean(1, keepdim=True))
                   .expand(-1, HW, -1)], -1)
    y, S = gelu(*linear(y, S, fc2a))
    y, S = gelu(*linear(y, S, fc2b))
    y, S = linear(y, S, fc2c)
    return y.squeeze(-1), S.squeeze(-1)


# (b, H, W, (Hc, Wc) or None, alpha_index)
PRED_CASES = [
    (1, 1, 1, None, 0), (3, 1, 1, (1, 1), 3),          # HW = 1: one tile, a 1 x 1 coarse level
    (3, 1, 7, (1, 1), 0), (8, 2, 4, (1, 3), 1),        # HW = 7, 8: one tile; H = 1; a 1 x n coarse level
    (1, 9, 1, (5, 1), 2), (3, 3, 3, (2, 2), 3),        # HW = 9: two tiles; W = 1
    (1, 7, 7, (4, 4), 1), (8, 13, 21, (7, 11), 2),     # HW = 49, 273 = 8k + 1: 7 and 35 tiles (odd)
    (3, 12, 10, (1, 5), 0), (1, 50, 81, (25, 41), 1),  # 15 and 507 tiles (odd), 1 x n coarse level
    (8, 16, 32, (8, 16), 3),                           # b h w = 4096, 64 tiles (even)
]


def _pred_tokens(b, HW, g):
    mem = torch.randn(b, HW, 256, generator=g)
    if HW > 2:
        mem[0, 1] = 3.25                                            # a constant row: LayerNorm gives beta
        mem[-1, HW - 1] = 1e4 + 1e-2 * torch.randn(256, generator=g)  # a large mean, a tiny spread
    return mem


def _run_predictor(pkg, mp, mem_lvl, H, W, coarse, ai, alpha, lead=5, tail=3, sentinel=None):
    """The level at token offset `lead` of a larger buffer, the coarse scores behind it -> (raw, level start)."""
    b, HW, _ = mem_lvl.shape
    Hc, Wc = coarse.shape[1:] if coarse is not None else (0, 0)
    nv = lead + HW + Hc * Wc + tail
    mem = torch.zeros(b, nv, 256)
    mem[:, lead:lead + HW] = mem_lvl
    raw = sentinel.clone() if sentinel is not None else torch.full((b, nv), -7.0)
    if coarse is not None:
        raw[:, lead + HW:lead + HW + Hc * Wc] = coarse.reshape(b, -1)
    raw = raw.to(DEV)
    cs = raw[:, lead + HW:lead + HW + Hc * Wc] if coarse is not None else None
    ln = mp.layer1[0]
    pkg.cabi.mask_predictor_level(mem.to(DEV), lead, H, W, cs, Hc, Wc, alpha.to(DEV), ai, ln.weight, ln.bias, ln.eps,
                                  *mp.transposed_weights(), raw, lead)
    return raw.cpu(), lead


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(PRED_CASES)))
def test_mask_predictor_level_vs_float64(pkg, case):
    """Within C_PRED of MaskPredictor in float64 on the float64 modulated tokens (a constant row, a row of mean 1e4 and
    standard deviation 1e-2); nothing outside the level's slice is written; a repeat gives the same bits."""
    b, H, W, hcwc, ai = PRED_CASES[case]
    g = torch.Generator().manual_seed(700 + case)
    mp = _predictor(70)
    mp64 = __import__("copy").deepcopy(mp).double()
    mp = mp.to(DEV)
    alpha = torch.tensor([0.3, -0.6, 1.1, -0.25])
    mem = _pred_tokens(b, H * W, g)
    coarse = torch.randn(b, *hcwc, generator=g) if hcwc else None
    raw, lead = _run_predictor(pkg, mp, mem, H, W, coarse, ai, alpha)
    if hcwc:
        m, E = modulate_ref(mem, coarse, float(alpha[ai]), H, W, *hcwc)
    else:
        m, E = mem.double(), torch.zeros(b, H * W, 256, dtype=torch.float64)
    with torch.no_grad():
        ref, S = predictor_ref(mp64, m, E)
        assert (mp64(m).squeeze(-1) - ref).abs().max() < 1e-9 * (1 + ref.abs().max())
    check_bound("mask_predictor_level", raw[:, lead:lead + H * W], ref, S, C_PRED)
    outside = torch.ones(raw.shape[1], dtype=torch.bool)
    outside[lead:lead + H * W] = False
    sentinel = torch.full_like(raw, -7.0)
    if coarse is not None:
        sentinel[:, lead + H * W:lead + H * W + coarse[0].numel()] = coarse.reshape(b, -1)
    assert same_bits(raw[:, outside], sentinel[:, outside])
    again, _ = _run_predictor(pkg, mp, mem, H, W, coarse, ai, alpha)
    assert same_bits(again, raw)


@pytest.mark.gpu
def test_mask_predictor_level_non_finite_token_stays_in_its_image(pkg):
    """A NaN or inf in one token makes its own image's level NaN (through the token mean); the other images keep the bits
    of the clean run."""
    mp = _predictor(71).to(DEV)
    alpha = torch.tensor([0.3, -0.6, 1.1, -0.25])
    g = torch.Generator().manual_seed(72)
    for b, H, W, hcwc in ((3, 7, 7, (4, 4)), (3, 1, 1, None), (8, 13, 21, (7, 11))):
        mem = torch.randn(b, H * W, 256, generator=g)
        coarse = torch.randn(b, *hcwc, generator=g) if hcwc else None
        clean, lead = _run_predictor(pkg, mp, mem, H, W, coarse, 1, alpha)
        for v in (float("nan"), float("inf")):
            bad = mem.clone()
            bad[1, H * W // 2, 77] = v
            got, _ = _run_predictor(pkg, mp, bad, H, W, coarse, 1, alpha)
            lvl = slice(lead, lead + H * W)
            assert torch.isnan(got[1, lvl]).all(), (b, H, W, v)
            keep = torch.arange(b) != 1
            assert same_bits(got[keep], clean[keep]) and same_bits(got[1, :lead], clean[1, :lead])


def score_loop_ref(mp64, mem, shapes, alpha, raw):
    """The score loop (salience_transformer.py salience_filter) in float64, level by level: each level modulated by the
    scores `raw` holds for the next coarser one, as the route under test computed them -> (raw, S)."""
    b = mem.shape[0]
    sizes = [h * w for h, w in shapes]
    starts = [sum(sizes[:i]) for i in range(len(shapes))]
    ref = torch.zeros(b, sum(sizes), dtype=torch.float64)
    S = torch.zeros_like(ref)
    for lvl in range(len(shapes) - 1, -1, -1):
        (h, w), s0 = shapes[lvl], starts[lvl]
        m = mem[:, s0:s0 + h * w].double()
        if lvl == len(shapes) - 1:
            E = torch.zeros_like(m)
        else:
            (hc, wc), s1 = shapes[lvl + 1], starts[lvl + 1]
            m, E = modulate_ref(m, raw[:, s1:s1 + hc * wc], float(alpha[lvl]), h, w, hc, wc)
        with torch.no_grad():
            ref[:, s0:s0 + h * w], S[:, s0:s0 + h * w] = predictor_ref(mp64, m, E)
    return ref, S


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [4096, 4097])
def test_score_loop_at_the_route_boundary(pkg, monkeypatch, rows):
    """b h w = 4096 takes the fused route, 4097 forward_fast: the levels each route ran are recorded (as routed, and with
    the fused route switched off), and each launch of the fused route is its two kernels.  Every level of both runs is
    within C_LOOP of MaskPredictor in float64 on the float64 modulation by the coarser scores that run computed."""
    import salience_detr_b200.salience_transformer as st
    shapes = {4096: [(64, 64), (32, 32), (16, 16), (8, 8)], 4097: [(17, 241), (9, 121), (5, 61), (3, 31)]}[rows]
    fused_want = {4096: {(64, 64), (32, 32), (16, 16), (8, 8)}, 4097: {(9, 121), (5, 61), (3, 31)}}[rows]
    model = _score_model(pkg)
    b, nv = 1, sum(h * w for h, w in shapes)
    masks = [torch.zeros(b, h, w, dtype=torch.bool, device=DEV) for h, w in shapes]
    plan = model.make_plan(masks)
    g = torch.Generator().manual_seed(rows)
    feat, lpos = torch.randn(b, nv, 256, generator=g).to(DEV), torch.randn(b, nv, 256, generator=g).to(DEV)
    fused, fast = [], []
    fused_call, fast_call = pkg.cabi.mask_predictor_level, model.enc_mask_predictor.forward_fast

    def record_fused(mem_all, level_start, H, W, *args):
        n0 = pkg.cabi.launch_count()
        out = fused_call(mem_all, level_start, H, W, *args)
        fused.append(((H, W), pkg.cabi.launch_count() - n0))
        return out

    def record_fast(m):
        fast.append(m.shape[1])
        return fast_call(m)

    monkeypatch.setattr(pkg.cabi, "mask_predictor_level", record_fused)
    monkeypatch.setattr(model.enc_mask_predictor, "forward_fast", record_fast)
    out = {}
    with torch.no_grad():
        x = (feat + lpos) * plan.keep
        mem = pkg.gemm.linear(x, model.enc_output.weight, model.enc_output.bias)
        mem = pkg.cabi.add_layernorm(mem, None, model.enc_output_norm.weight, model.enc_output_norm.bias,
                                     model.enc_output_norm.eps)
        for small in (st.PREDICTOR_SMALL_ROWS, 0):
            fused.clear()
            fast.clear()
            with monkeypatch.context() as mc:
                mc.setattr(st, "PREDICTOR_SMALL_ROWS", small)
                out[small] = model.salience_filter(feat, lpos, plan)[0].cpu()
            fused_hw = {hw for hw, _ in fused}
            if small:
                assert fused_hw == fused_want and len(fused) == len(fused_want) and all(n == 2 for _, n in fused)
                assert sorted(fast) == sorted(h * w for h, w in shapes if (h, w) not in fused_want)
            else:
                assert not fused and sorted(fast) == sorted(h * w for h, w in shapes)
    mp64 = __import__("copy").deepcopy(model.enc_mask_predictor).cpu().double()
    for small, raw in out.items():
        ref, S = score_loop_ref(mp64, mem.cpu(), shapes, model.alpha.detach().cpu(), raw)
        check_bound("score_loop", raw, ref, S, C_LOOP)


def _score_model(pkg):
    from salience_detr_b200.synthetic import build_model
    model = build_model(layers=1)
    g = torch.Generator().manual_seed(90)
    with torch.no_grad():
        mp = model.enc_mask_predictor
        for p in mp.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.08 if p.dim() > 1 else 0.2))
        mp.layer1[0].weight.add_(1.0)
        model.alpha.copy_(torch.tensor([0.4, -0.7, 0.9]))
    return model.to(DEV)


# ==== 4. mask_plan and sine_pos_tokens ==================================================================================
def _plan_model():
    from salience_detr_b200.synthetic import build_model
    return build_model(layers=1)


def norm_coords(masks, offset=-0.5, eps=1e-6, scale=2 * math.pi):
    """PositionEmbeddingSine(normalize=True)'s normalised coordinates in float32 torch ops (position_encoding.py:48-56)
    -> (ynorm, xnorm) (b, Nv)."""
    ys, xs = [], []
    for m in masks:
        nm = (~m).to(torch.float32)
        y, x = nm.cumsum(1, dtype=torch.float32), nm.cumsum(2, dtype=torch.float32)
        y = (y + offset) / (y[:, -1:, :] + eps) * scale
        x = (x + offset) / (x[:, :, -1:] + eps) * scale
        ys.append(y.flatten(1))
        xs.append(x.flatten(1))
    return torch.cat(ys, 1), torch.cat(xs, 1)


def _plan_masks(shapes, b, seed, pad_first_row=None, pad_first_col=None):
    g = torch.Generator().manual_seed(seed)
    masks = []
    for l, (h, w) in enumerate(shapes):
        m = torch.rand(b, h, w, generator=g) < 0.25                     # random holes
        m[0, :, w - w // 5:] = True                                     # right padding
        m[b - 1, h - h // 4:, :] = True                                 # bottom padding
        if pad_first_row == l:
            m[0, 0, :] = True                                           # vw = 0
        if pad_first_col == l:
            m[b - 1, :, 0] = True                                       # vh = 0
        masks.append(m)
    return masks


# (level shapes, level with a fully padded first row in image 0, level with a fully padded first column in the last image)
PLAN_CASES = [
    ([(7, 300), (300, 5), (1, 37), (23, 1)], None, None),    # 300 wide, 300 tall, 1 x N, N x 1
    ([(260, 270), (1, 300), (300, 1), (2, 2)], 0, 3),       # both scans strided over 256 threads; vh = 0, vw = 0
    ([(40, 60), (20, 30), (10, 15), (5, 8)], 1, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(PLAN_CASES)))
def test_mask_plan_vs_torch(pkg, case):
    """make_plan on the device against make_plan on the CPU (focus budgets, valid ratios, keep) exactly, the valid counts
    exactly, ynorm / xnorm against the float32 torch chain bit for bit."""
    shapes, row, col = PLAN_CASES[case]
    masks = _plan_masks(shapes, 2, 800 + case, row, col)
    if row is not None:
        assert not (~masks[row][0, 0]).any()
    model = _plan_model()
    want = model.make_plan(masks)
    gpu_model = model.to(DEV)
    got = gpu_model.make_plan([m.to(DEV) for m in masks])
    assert got.level_token_nums == want.level_token_nums and got.focus_host == want.focus_host
    assert torch.equal(got.focus_token_nums.cpu(), want.focus_token_nums)
    assert torch.equal(got.valid_ratios.cpu(), want.valid_ratios)
    assert torch.equal(got.keep.cpu(), want.keep)
    starts = [sum(h * w for h, w in shapes[:l]) for l in range(len(shapes) + 1)]
    for l, i in ((row, 0), (col, 1)):  # a valid size of 0: ratio 0, nothing of the level kept
        if l is not None:
            assert float(want.valid_ratios[i, l, 0 if l == row else 1]) == 0.0
            assert not want.keep[i, starts[l]:starts[l + 1]].any()
    mp = pkg.cabi.mask_plan(flatten_levels(masks).to(torch.uint8).to(DEV), shapes, [0.4, 0.8, 1.0, 1.0])
    valid = torch.stack([(~m).sum((1, 2)) for m in masks], -1).to(torch.int32)
    assert torch.equal(mp["valid"].cpu(), valid)
    yn, xn = norm_coords(masks)
    assert same_bits(mp["ynorm"], yn) and same_bits(mp["xnorm"], xn)
    assert same_bits(got.scratch["ynorm"], yn) and same_bits(got.scratch["xnorm"], xn)


def test_mask_plan_cases_reach_the_edges():
    """The table has levels wider and taller than the 256 threads of a scan, 1 x N and N x 1 levels, and levels whose
    valid height or width is 0."""
    shapes = [s for c in PLAN_CASES for s in c[0]]
    assert any(w > 256 for _, w in shapes) and any(h > 256 for h, _ in shapes)
    assert any(h == 1 and w > 1 for h, w in shapes) and any(w == 1 and h > 1 for h, w in shapes)
    for shapes, row, col in PLAN_CASES:
        masks = _plan_masks(shapes, 2, 0, row, col)
        if row is not None:
            assert int((~masks[row][0, 0, :]).sum()) == 0
        if col is not None:
            assert int((~masks[col][1, :, 0]).sum()) == 0
    assert any(c[1] is not None for c in PLAN_CASES) and any(c[2] is not None for c in PLAN_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("npf", [4, 64, 128, 132])
def test_sine_pos_tokens_vs_float64(pkg, npf):
    """sin / cos of e / dim_t within C_SINE u (1 + |e / dim_t|) of float64 (the float32 division's rounding and sinf's),
    channel order [y sin, y cos, ... | x sin, x cos, ...], 1003 rows (not a multiple of the 8 rows of a CTA), coordinates from
    a real mask plan plus the padded columns' large values."""
    shapes = [(7, 300), (300, 5), (1, 37), (23, 1)]
    masks = _plan_masks(shapes, 2, 9, 0, 3)
    mp = pkg.cabi.mask_plan(flatten_levels(masks).to(torch.uint8).to(DEV), shapes, [1.0] * 4)
    yn, xn = mp["ynorm"].reshape(-1)[:1003].view(1, -1), mp["xnorm"].reshape(-1)[-1003:].view(1, -1)
    yn, xn = yn.contiguous(), xn.contiguous()
    dim_t = 10000 ** (2 * torch.arange(npf).div(2, rounding_mode="floor") / npf)
    dim_tx = (20 ** (2 * torch.arange(npf).div(2, rounding_mode="floor") / npf)).float()
    dim_ty = dim_t.float()
    got = pkg.cabi.sine_pos_tokens(yn, xn, dim_ty.to(DEV), dim_tx.to(DEV)).cpu()
    assert got.shape == (1, 1003, 2 * npf)
    parts, scales = [], []
    for e, dt in ((yn.cpu(), dim_ty), (xn.cpu(), dim_tx)):
        arg = e.double()[..., None] / dt.double()
        parts.append(torch.where(torch.arange(npf) % 2 == 0, torch.sin(arg), torch.cos(arg)))
        scales.append(1 + arg.abs())
    check_bound("sine_pos_tokens", got, torch.cat(parts, -1), torch.cat(scales, -1), C_SINE)
    assert yn.abs().max() > 1e5  # the padded columns' coordinates reach large arguments


# ==== 5. salience_targets ===============================================================================================
LIMITS = ((-1, 64), (64, 128), (128, 256), (256, 99999))


def targets_f32(boxes, num_boxes, shapes, strides, limits):
    """The kernel's arithmetic in float32 torch ops (salience_detr.py:64-114 at noise 0), padding rows unread; also the
    (mn == 0, mx == lo, mx == hi) edge counts -> (targets (b, Nv), edges)."""
    out, edges = [], [0, 0, 0]
    for i in range(boxes.shape[0]):
        bx = boxes[i, :int(num_boxes[i])]
        row = []
        for (h, w), (sy, sx), (lo, hi) in zip(shapes, strides, limits):
            ys = (torch.arange(h, dtype=torch.float32) + 0.5) * torch.tensor(sy, dtype=torch.float32)
            xs = (torch.arange(w, dtype=torch.float32) + 0.5) * torch.tensor(sx, dtype=torch.float32)
            cy, cx = [t.reshape(-1, 1) for t in torch.meshgrid(ys, xs, indexing="ij")]
            if bx.shape[0] == 0:
                row.append(torch.zeros(h * w))
                continue
            dl, dt, dr, db = cx - bx[:, 0], cy - bx[:, 1], bx[:, 2] - cx, bx[:, 3] - cy
            d = torch.stack([dl, dt, dr, db], -1)
            mn, mx = d.amin(-1), d.amax(-1)
            lo32, hi32 = torch.tensor(lo, dtype=torch.float32), torch.tensor(hi, dtype=torch.float32)
            inside = mn > 0
            edges[0] += int((mn == 0).sum())
            edges[1] += int((inside & (mx == lo32)).sum())
            edges[2] += int((inside & (mx == hi32)).sum())
            pos = (inside & (mx > lo32) & (mx <= hi32)).any(-1)
            ddx, ddy = (dl - dr) / (dl + dr), (dt - db) / (dt + db)
            conf = 1 - torch.sqrt(ddx * ddx + ddy * ddy) / 2
            best = torch.where(inside, conf, torch.zeros_like(conf)).amax(-1).clamp_min(0)
            row.append(torch.where(pos, best, torch.zeros_like(best)))
        out.append(torch.cat(row))
    return torch.stack(out), edges


def targets_f64(boxes, num_boxes, shapes, strides, limits, decide):
    """The centredness in float64 from the same distances, where the float32 restatement `decide` is positive."""
    out = []
    for i in range(boxes.shape[0]):
        bx = boxes[i, :int(num_boxes[i])].double()
        row = []
        for (h, w), (sy, sx) in zip(shapes, strides):
            ys = ((torch.arange(h, dtype=torch.float32) + 0.5) * torch.tensor(sy, dtype=torch.float32)).double()
            xs = ((torch.arange(w, dtype=torch.float32) + 0.5) * torch.tensor(sx, dtype=torch.float32)).double()
            cy, cx = [t.reshape(-1, 1) for t in torch.meshgrid(ys, xs, indexing="ij")]
            if bx.shape[0] == 0:
                row.append(torch.zeros(h * w, dtype=torch.float64))
                continue
            dl, dt, dr, db = cx - bx[:, 0], cy - bx[:, 1], bx[:, 2] - cx, bx[:, 3] - cy
            inside = torch.stack([dl, dt, dr, db], -1).amin(-1) > 0
            conf = 1 - torch.sqrt(((dl - dr) / (dl + dr)) ** 2 + ((dt - db) / (dt + db)) ** 2) / 2
            row.append(torch.where(inside, conf, torch.zeros_like(conf)).amax(-1).clamp_min(0))
        out.append(torch.cat(row))
    return torch.where(decide > 0, torch.stack(out), torch.zeros(1, dtype=torch.float64))


TGT_SHAPES = [(25, 38), (13, 19), (7, 10), (4, 5)]
TGT_STRIDES = [(8.0, 8.0), (16.0, 16.0), (32.0, 32.0), (64.0, 64.0)]


def edge_boxes():
    """Boxes whose sides pass through pixel centres ((x + 1/2) s) and whose largest border distance from a centre is exactly
    a level's lo or hi: centres on an edge (mn = 0), mx = lo (excluded) and mx = hi (included)."""
    out = []
    for (sy, sx), (lo, hi) in zip(TGT_STRIDES, LIMITS):
        if lo < 0:
            lo = 40
        hi = min(hi, 256 + 24)
        cx, cy = 4.5 * sx, 2.5 * sy  # a pixel centre of the level
        out += [[cx - lo, cy - 2, cx + 3, cy + 2],     # mx = lo at (cx, cy)
                [cx - 3, cy - hi, cx + 4, cy + 1],     # mx = hi at (cx, cy)
                [cx, cy - 10, cx + 2 * sx, cy + 10],   # left side through a centre column
                [cx - sx, cy, cx + sx, cy + 3 * sy]]   # top side through a centre row
    return torch.tensor(out, dtype=torch.float32)


@pytest.mark.gpu
def test_salience_targets_vs_float32_and_float64(pkg):
    """Bit for bit against the float32 restatement and within C_TGT of float64: random boxes, boxes on pixel centres and on
    the level limits, an image without boxes, max_boxes = 0.  Rows past num_boxes[b] hold NaN boxes and boxes that would
    change every image's targets if they were read (checked on the restatement): the result is the one of the first
    num_boxes[b] rows."""
    g = torch.Generator().manual_seed(13)
    edge = edge_boxes()
    rnd = torch.rand(40, 2, generator=g) * 300
    rand = torch.cat([rnd, rnd + torch.rand(40, 2, generator=g) * 300 + 1], -1)
    mb = 48
    boxes = torch.full((4, mb, 4), float("nan"))
    num = torch.tensor([edge.shape[0], 40, 0, 7], dtype=torch.int32)
    boxes[0, :edge.shape[0]] = edge
    boxes[1, :40] = rand
    boxes[3, :7] = rand[:7] + 0.25
    # padding rows that matter if read: boxes of levels 0 and 1 around many pixel centres (largest border distance of the
    # central pixels about 30 and about 80 px), after a NaN row
    poison = torch.tensor([[40.0, 40.0, 100.0, 90.0], [100.0, 100.0, 260.0, 220.0], [20.0, 130.0, 190.0, 280.0]])
    for i in range(4):
        n = int(num[i])
        boxes[i, n + 1:n + 1 + poison.shape[0]] = poison
    want, edges = targets_f32(boxes, num, TGT_SHAPES, TGT_STRIDES, LIMITS)
    assert all(e > 0 for e in edges), edges
    assert (want[0] > 0).any() and (want[1] > 0).any() and not want[2].any()
    read_all, _ = targets_f32(boxes, torch.full((4,), mb, dtype=torch.int32), TGT_SHAPES, TGT_STRIDES, LIMITS)
    assert all(not torch.equal(read_all[i], want[i]) for i in range(4))  # reading a padding row would show
    got = pkg.cabi.salience_targets(boxes.to(DEV), num.to(DEV), TGT_SHAPES, TGT_STRIDES, LIMITS)
    assert same_bits(got, want)
    ref = targets_f64(boxes, num, TGT_SHAPES, TGT_STRIDES, LIMITS, want)
    check_bound("salience_targets", got, ref, torch.ones_like(ref), C_TGT)
    empty = pkg.cabi.salience_targets(torch.zeros(2, 0, 4, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV),
                                      TGT_SHAPES, TGT_STRIDES, LIMITS)
    assert same_bits(empty, torch.zeros(2, sum(h * w for h, w in TGT_SHAPES)))
