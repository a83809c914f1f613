"""The token-layout convolutions (csrc/neck.cu) and the ResNet front end (csrc/backbone.cu) on every launch path, against
float64 F.conv2d, its autograd and torch's pooling / interpolation.

Kernels: `sdetr_conv2d_f16x3` (forward, bias, residual z that may alias y, none / ReLU / SiLU), `_dgrad` (stride 1: the
forward kernel on flipped weights; stride 2: the transposed mode), `_wgrad` (the pixel range split by the shape, the
splits summed in order, optional cout_scale), `_split_weight`, `sdetr_context_gate`, `sdetr_upsample_nearest_concat` and
its backward, `sdetr_resnet_stem`, `sdetr_maxpool3x3s2_tokens` and `sdetr_frozen_bn_fold`.

Case table: (k, stride) in {1, 3} x {1, 2}; (Cin, Cout, groups) in CHANNELS, three of them with Cout / groups != Cin /
groups; the maps 1x1, 1x7, 7x1, 2x3, 4x6, 13x21, 25x42 and six maps whose last 64-pixel tile holds 1, 63 or 64 rows; b in
{1, 2}; and the 800x1333 layers of ResNet-50, the neck and the ChannelMapper, each once.  The CPU tests restate the
launch arithmetic and assert the table reaches every edge: last tiles of 1, 63 and 64 rows, M < 64, one wgrad split,
one k-block per split, a short last split, every (H mod 2, W mod 2) at stride 2 for k = 1 and 3, and context-gate chunk
counts of 1, 2 and many with a partial last chunk.

Every operand is a view into a NaN-filled buffer: a level slice with NaN rows before and after it, and a row stride four
channels wider than the operand, with NaN in the extra channels.  The outputs are written into NaN-filled buffers whose
rows and channels outside the view must come back with the same bits.  pow2_scale ignores non-finite entries, so the
scales are taken over the whole fenced buffer; a read outside an operand shows up as a NaN in the result.

Non-finite locality: `receptive_fields_x` and `receptive_fields_dy` give, for a non-finite input or output-gradient element, the exact set of
forward outputs, input-gradient entries and weight-gradient entries that must become non-finite, group by group.  A CPU
test checks it against float64 F.conv2d and its gradients holding one NaN; the GPU tests use it as the oracle, and every
entry outside it must keep the clean run's bits.

Bounds are |got - ref| <= c * (2^-24 * S + T) element-wise.  S is the float64 result on absolute values (|x| conv |w|,
plus |bias| and |z|).  T covers the fp16 subnormal range of the split: a lo part (or a whole operand) below 2^-14 of the
scaled range is rounded to the subnormal spacing 2^-24, an absolute error of at most 2^-25 in scaled units, so T is
2^-25 / a_scale * (sum of |w| over the window) + 2^-25 / w_scale * (sum of |x| over the window).  SiLU adds its slope
(below 1.1) and four roundings of its own result (expf, the add, the division).  SDETR_CONV_OBSERVE=1 prints the largest
c each bound needed."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import salience_detr_b200 as pkg

cabi = pkg.cabi
gpu = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24  # unit round-off of float32
NAN = float("nan")
KCV = 64            # conv tile: 64 output pixels x 64 output channels, k-blocks of 64 channels
WG_TARGET_CTAS = 512
GATE_CHUNK = 128

# Bound constants c of |got - ref| <= c (2^-24 S + T).  Each is about four times the largest c observed over every case of
# this file on an H100 80GB HBM3 at 700 W (noted beside it).
C_FWD = 68.0     # forward (observed 17.0 over the case table, 3.02 at the real layer shapes)
C_DGRAD = 75.0   # input gradient (observed 18.6, 4.92)
C_WGRAD = 80.0   # weight gradient (observed 20.2, 2.02; 3.72 over the split cases)
C_GATE = 4.0     # context gate (observed 1.03)
C_UPS = 10.0     # upsample backward against float64 (observed 2.55)
C_STEM = 23.0    # ResNet stem (observed 5.67)
# The 2^-17 S bound of the older tests is c = 128: about six times the largest c any convolution path needed.

OBSERVED = {}


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    if os.environ.get("SDETR_CONV_OBSERVE"):
        print("\nOBSERVED", {k: float(f"{v:.3g}") for k, v in sorted(OBSERVED.items())})


def check_bound(name, got, ref, S, T, c):
    """|got - ref| <= c (u S + T) element-wise (NaN anywhere fails); records the c the case needed"""
    got = got.double().to(ref.device)
    err = (got - ref).abs()
    den = U * S + T
    need = (err / den.clamp_min(1e-300)).masked_fill((den == 0) & (err == 0), 0)
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(need.max()) if need.numel() else 0.0)
    bad = ~(err <= c * den)
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} of {bad.numel()} outside c={c} (needs {float(need.max()):.3g})"


# ==== host restatement of the launch arithmetic ===========================================================================
def conv_out(h, w, k, s):
    pad = k // 2
    return (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1


def conv_grid(b, h, w, cout, k, s):
    """(grid.x, grid.y, M, rows of the last 64-pixel tile) of sdetr_conv2d_f16x3"""
    ho, wo = conv_out(h, w, k, s)
    m = b * ho * wo
    return -(-m // KCV), cout // KCV, m, m - (-(-m // KCV) - 1) * KCV


def dgrad_grid(b, h, w, cin, k, s):
    """(grid.x, grid.y, M, rows of the last tile) of sdetr_conv2d_f16x3_dgrad: one output pixel per input pixel of the forward"""
    m = b * h * w
    return -(-m // KCV), cin // KCV, m, m - (-(-m // KCV) - 1) * KCV


def wgrad_splits(m, tiles):
    """(splits, k-blocks per split, k-blocks) of the weight gradient's pixel range: a function of the shape alone"""
    kblocks = -(-m // KCV)
    if kblocks == 0:
        return 0, 1, 0
    want = min(max(-(-WG_TARGET_CTAS // tiles), 1), kblocks)
    per = -(-kblocks // want)
    return -(-kblocks // per), per, kblocks


def wgrad_tiles(cin, cout, groups, k):
    return (cout // KCV) * ((cin // groups) // KCV) * k * k


def wgrad_workspace_floats(b, ho, wo, cin, cout, groups, k):
    splits, _, _ = wgrad_splits(b * ho * wo, wgrad_tiles(cin, cout, groups, k))
    return splits * cout * (cin // groups) * k * k


def gate_chunks(hw):
    """(chunks, pixels of the last chunk) of the context gate"""
    n = -(-hw // GATE_CHUNK)
    return n, hw - (n - 1) * GATE_CHUNK


def gate_workspace_floats(b, hw, c):
    return b * gate_chunks(hw)[0] * (c + 2) + b * c


# ==== the case table ======================================================================================================
KS = [(1, 1), (1, 2), (3, 1), (3, 2)]
# (Cin, Cout, groups): the last three have Cout / groups != Cin / groups
CHANNELS = [(64, 64, 1), (256, 256, 4), (512, 256, 1), (128, 64, 1), (2048, 256, 1), (256, 512, 4), (256, 512, 2),
            (512, 256, 4)]
MAPS = [(1, 1), (1, 7), (7, 1), (2, 3), (4, 6), (13, 21), (25, 42)]
# maps whose last 64-pixel tile (b = 1) holds 1, 63 or 64 rows: stride 1 (5x13, 1x127, 8x8) and stride 2 (9x25, 1x253, 16x16)
TILE_MAPS = [(5, 13), (1, 127), (8, 8), (9, 25), (1, 253), (16, 16)]
FAMILIES = ["normal", "small", "large", "decades", "spike", "zeros", "allzero", "wdecades"]
ACTS = [0, cabi.ACT_RELU, cabi.ACT_SILU]
ZMODES = ["none", "sep", "alias"]
DMODES = ["none", "z", "z_alias", "m", "z_m_alias"]


def conv_cases(k, s, ch):
    """the maps of one (k, stride, channels) entry, each with its batch and variant (act, bias, z, value family)"""
    ci = CHANNELS.index(ch)
    out = []
    for i, hw in enumerate(MAPS + TILE_MAPS):
        j = i + 5 * ci + 3 * KS.index((k, s))
        b = 1 if hw in TILE_MAPS else 1 + j % 2
        out.append(dict(hw=hw, b=b, act=ACTS[j % 3], bias=(j // 3) % 2 == 0, z=ZMODES[(j // 6) % 3], fam=FAMILIES[j % 8],
                        dmode=DMODES[j % 5], dfam=FAMILIES[(j + 1) % 6]))
    return out


TABLE = [(k, s, ch) for k, s in KS for ch in CHANNELS]
TABLE_IDS = [f"k{k}s{s}_{ci}-{co}g{g}" for k, s, (ci, co, g) in TABLE]

# 800x1333, bs = 2: name -> (k, stride, Cin, Cout, groups, H, W)
REAL = {
    "r50_layer2_conv2": (3, 2, 128, 128, 1, 200, 334),
    "r50_layer2_down": (1, 2, 256, 512, 1, 200, 334),
    "r50_layer3_conv2": (3, 2, 256, 256, 1, 100, 167),
    "r50_layer3_down": (1, 2, 512, 1024, 1, 100, 167),
    "r50_layer4_conv2": (3, 2, 512, 512, 1, 50, 84),
    "r50_layer4_down": (1, 2, 1024, 2048, 1, 50, 84),
    "neck_3x3_g4": (3, 1, 256, 256, 4, 100, 168),
    "mapper_1x1_512": (1, 1, 512, 256, 1, 100, 167),
    "mapper_1x1_1024": (1, 1, 1024, 256, 1, 50, 84),
    "mapper_1x1_2048": (1, 1, 2048, 256, 1, 25, 42),
    "mapper_extra_3x3s2": (3, 2, 2048, 256, 1, 25, 42),
}

# weight-gradient split cases: name -> (k, stride, Cin, Cout, groups, H, W, b)
WGRAD_SPLITS = {
    "one_split_big_tiles": (3, 1, 2048, 256, 1, 13, 21, 2),    # 1152 tiles: one split of 9 k-blocks
    "one_split_one_kblock": (1, 1, 64, 64, 1, 5, 12, 1),       # M = 60: one k-block
    "per1": (1, 1, 64, 64, 1, 13, 21, 2),                      # 9 k-blocks, 9 splits of one
    "short_last": (3, 1, 64, 64, 1, 100, 168, 2),              # 525 k-blocks, 53 splits of 10, the last of 5
    "short_last_s2": (3, 2, 256, 256, 4, 100, 167, 2),         # 36 tiles, 132 k-blocks, 15 splits of 9, the last of 6
    "several_g4": (3, 1, 256, 512, 4, 25, 42, 2),              # 72 tiles, 33 k-blocks, 7 splits of 5, the last of 3
}

GATE_CASES = [  # (HW, b, R, z)
    (1, 1, 1, False), (127, 2, 16, True), (128, 8, 256, False), (129, 2, 1, True), (255, 1, 16, False),
    (257, 8, 16, True), (16800, 2, 16, False), (16800, 1, 256, True), (257, 2, 256, False), (128, 1, 1, True),
]
UPS_CASES = [((13, 21), (26, 42)), ((13, 21), (25, 42)), ((7, 11), (20, 30)), ((1, 1), (3, 5)), ((9, 10), (9, 10)),
             ((25, 42), (13, 21)), ((7, 20), (3, 7)), ((50, 84), (100, 168))]


# ==== receptive fields ====================================================================================================
def receptive_fields_x(shape, n, y, x, c):
    """for a non-finite x[n, y, x, c] of the convolution shape (b, H, W, Cin, Cout, groups, k, stride): (forward outputs
    (b, Ho, Wo, Cout), weight-gradient entries (Cout, Cin / groups, k, k)) that must become non-finite"""
    b, H, W, cin, cout, groups, k, s = shape
    ho, wo = conv_out(H, W, k, s)
    cin_g, cout_g, pad = cin // groups, cout // groups, k // 2
    g = c // cin_g
    fwd = torch.zeros(b, ho, wo, cout, dtype=torch.bool)
    wg = torch.zeros(cout, cin_g, k, k, dtype=torch.bool)
    for ky in range(k):
        for kx in range(k):
            oy, ox = y + pad - ky, x + pad - kx
            if oy % s or ox % s or not (0 <= oy // s < ho and 0 <= ox // s < wo):
                continue
            fwd[n, oy // s, ox // s, g * cout_g:(g + 1) * cout_g] = True
            wg[g * cout_g:(g + 1) * cout_g, c - g * cin_g, ky, kx] = True
    return fwd, wg


def receptive_fields_dy(shape, n, oy, ox, co):
    """for a non-finite dY[n, oy, ox, co]: (input-gradient entries (b, H, W, Cin), weight-gradient entries (Cout, Cin / groups,
    k, k)).  Every weight entry of row co changes: each tap multiplies dY by an input value, or by the zero of the padding."""
    b, H, W, cin, cout, groups, k, s = shape
    cin_g, cout_g, pad = cin // groups, cout // groups, k // 2
    g = co // cout_g
    dx = torch.zeros(b, H, W, cin, dtype=torch.bool)
    for ky in range(k):
        for kx in range(k):
            y, x = oy * s - pad + ky, ox * s - pad + kx
            if 0 <= y < H and 0 <= x < W:
                dx[n, y, x, g * cin_g:(g + 1) * cin_g] = True
    wg = torch.zeros(cout, cin_g, k, k, dtype=torch.bool)
    wg[co] = True
    return dx, wg


def dgrad_weight(w, groups):
    """(Cout, Cin / groups, k, k) -> the (Cin, k, k, Cout / groups) input-gradient weight: flipped in both spatial axes and
    transposed per group"""
    cout, cin_g, k, _ = w.shape
    return w.reshape(groups, cout // groups, cin_g, k, k).flip(3, 4).permute(0, 2, 3, 4, 1).reshape(groups * cin_g, k, k,
                                                                                                   cout // groups)


def nchw(t, hw):
    b, _, c = t.shape
    return t.transpose(1, 2).reshape(b, c, *hw)


def tok(t):
    return t.flatten(2).transpose(1, 2)


# ==== CPU tests ===========================================================================================================
def test_launch_arithmetic_matches_library_and_torch():
    import __graft_entry__ as entry
    entry.build()
    lib = cabi.lib()
    for h, w in MAPS + TILE_MAPS + [(200, 334), (100, 167), (50, 84), (25, 42), (800, 1333)]:
        for k, s in KS:
            ref = F.conv2d(torch.zeros(1, 1, h, w), torch.zeros(1, 1, k, k), None, s, k // 2).shape[2:]
            assert conv_out(h, w, k, s) == tuple(ref)
    for k, s, (cin, cout, g) in TABLE:
        for case in conv_cases(k, s, (cin, cout, g)):
            ho, wo = conv_out(*case["hw"], k, s)
            assert lib.sdetr_conv2d_f16x3_wgrad_workspace_floats(case["b"], ho, wo, cin, cout, g, k) == \
                wgrad_workspace_floats(case["b"], ho, wo, cin, cout, g, k)
    for k, s, cin, cout, g, h, w, *b in list(WGRAD_SPLITS.values()) + [v + (2,) for v in REAL.values()]:
        ho, wo = conv_out(h, w, k, s)
        assert lib.sdetr_conv2d_f16x3_wgrad_workspace_floats(b[0], ho, wo, cin, cout, g, k) == \
            wgrad_workspace_floats(b[0], ho, wo, cin, cout, g, k)
    for hw, b, _, _ in GATE_CASES:
        assert lib.sdetr_context_gate_workspace_floats(b, hw, 256) == gate_workspace_floats(b, hw, 256)


def test_case_table_reaches_every_edge():
    last_tiles, small_m, parities = set(), False, set()
    variants, fams, dmodes = set(), set(), set()
    for k, s, ch in TABLE:
        for case in conv_cases(k, s, ch):
            (h, w), b = case["hw"], case["b"]
            _, _, m, last = conv_grid(b, h, w, ch[1], k, s)
            last_tiles.add(last)
            small_m |= m < KCV
            last_tiles.add(dgrad_grid(b, h, w, ch[0], k, s)[3])
            if s == 2:
                parities.add((k, h % 2, w % 2))
            variants.add((case["act"], case["bias"], case["z"]))
            fams.add(case["fam"])
            dmodes.add(case["dmode"])
    assert {1, 63, 64} <= last_tiles and small_m
    assert parities >= {(k, a, c) for k in (1, 3) for a in (0, 1) for c in (0, 1)}
    assert {(1, 7), (7, 1), (1, 1)} <= {c["hw"] for c in conv_cases(1, 2, CHANNELS[0])}  # H = 1 and W = 1
    assert len(variants) == 3 * 2 * 3 and set(FAMILIES) == fams and set(DMODES) == dmodes
    assert {ch for ch in CHANNELS if ch[2] > 1 and ch[1] // ch[2] == 2 * (ch[0] // ch[2])}
    # weight-gradient splits: one split, one k-block per split, a short last split
    seen = set()
    for k, s, cin, cout, g, h, w, b in WGRAD_SPLITS.values():
        splits, per, kblocks = wgrad_splits(b * conv_out(h, w, k, s)[0] * conv_out(h, w, k, s)[1], wgrad_tiles(cin, cout, g, k))
        seen |= {"one"} if splits == 1 else set()
        seen |= {"per1"} if per == 1 and splits > 1 else set()
        seen |= {"short"} if kblocks % per else set()
        seen |= {"one_kblock"} if kblocks == 1 else set()
    assert seen == {"one", "per1", "short", "one_kblock"}
    # context gate: 1, 2 and many chunks, full and partial last chunks
    chunks = {gate_chunks(hw) for hw, _, _, _ in GATE_CASES}
    assert {n for n, _ in chunks} >= {1, 2, 3, 132}
    assert any(n > 2 and last < GATE_CHUNK for n, last in chunks) and any(last == GATE_CHUNK for _, last in chunks)
    assert any(last == 1 for _, last in chunks)


SITES = [(0, 0, 0), (1, -1, -1), (0, 1, -1), (1, -1, 2), (0, 2, 3)]  # (n, y, x), negative from the far edge


@pytest.mark.parametrize("k,s", KS)
@pytest.mark.parametrize("groups,cin,cout", [(1, 4, 6), (2, 4, 8), (2, 6, 4)])
@pytest.mark.parametrize("hw", [(1, 1), (1, 6), (7, 1), (4, 6), (5, 7), (6, 5)])
def test_receptive_fields_match_float64_conv(k, s, groups, cin, cout, hw):
    """receptive_fields_* against float64 F.conv2d, its input gradient and its weight gradient on a CPU tensor holding one
    NaN, at every site of SITES that exists in the map and at the first and last channel"""
    b, (H, W) = 2, hw
    shape = (b, H, W, cin, cout, groups, k, s)
    ho, wo = conv_out(H, W, k, s)
    gen = torch.Generator().manual_seed(k + 7 * s + 31 * H + W + cin)
    w = torch.randn(cout, cin // groups, k, k, dtype=torch.float64, generator=gen)
    for n, y, x in SITES:
        for c in (0, cin - 1):
            if y >= H or x >= W or -y > H or -x > W:
                continue
            yy, xx = y % H, x % W
            xt = torch.randn(b, cin, H, W, dtype=torch.float64, generator=gen)
            xt[n, c, yy, xx] = NAN
            dy = torch.randn(b, cout, ho, wo, dtype=torch.float64, generator=gen)
            fwd, wg = receptive_fields_x(shape, n, yy, xx, c)
            assert torch.equal(~F.conv2d(xt, w, None, s, k // 2, groups=groups).isfinite(), fwd.permute(0, 3, 1, 2))
            got = torch.nn.grad.conv2d_weight(xt, w.shape, dy, s, k // 2, groups=groups)
            assert torch.equal(~got.isfinite(), wg)
            oy, ox = (y % ho, x % wo) if -y <= ho and -x <= wo and y < ho and x < wo else (0, 0)
            co = c * cout // cin
            xt = torch.randn(b, cin, H, W, dtype=torch.float64, generator=gen)
            dy[n, co, oy, ox] = NAN
            dxm, wgm = receptive_fields_dy(shape, n, oy, ox, co)
            got = torch.nn.grad.conv2d_input(xt.shape, w, dy, s, k // 2, groups=groups)
            assert torch.equal(~got.isfinite(), dxm.permute(0, 3, 1, 2))
            got = torch.nn.grad.conv2d_weight(xt, w.shape, dy, s, k // 2, groups=groups)
            assert torch.equal(~got.isfinite(), wgm)


def nearest_src(dst, n_in, n_out):
    """torch's nearest index rule in float32: min(floor(dst * (float)in / out), in - 1)"""
    scale = np.float32(n_in) / np.float32(n_out)
    return np.minimum(np.floor(np.asarray(dst, np.float32) * scale).astype(np.int64), n_in - 1)


def nearest_first_dst(n_in, n_out):
    """first destination of every source (and of n_in): the bounds of the backward's [first_dst(s), first_dst(s + 1)) ranges"""
    src = nearest_src(np.arange(n_out), n_in, n_out)
    return np.searchsorted(src, np.arange(n_in + 1), side="left")


@pytest.mark.parametrize("src,dst", UPS_CASES)
def test_nearest_restatement_matches_interpolate(src, dst):
    x = torch.arange(src[0] * src[1], dtype=torch.float32).view(1, 1, *src)
    up = F.interpolate(x, size=dst, mode="nearest")[0, 0].long()
    iy, ix = nearest_src(np.arange(dst[0]), src[0], dst[0]), nearest_src(np.arange(dst[1]), src[1], dst[1])
    assert torch.equal(up, torch.from_numpy(iy[:, None] * src[1] + ix[None, :]))
    fy = nearest_first_dst(src[0], dst[0])
    assert fy[0] == 0 and fy[-1] == dst[0] and (np.diff(fy) >= 0).all()
    if dst[0] < src[0]:
        assert (np.diff(fy) == 0).any()  # some sources receive no gradient


# ==== GPU helpers =========================================================================================================
def fenced(b, rows, c, data=None, pre=3, post=2, extra=4):
    """(view, buffer): a (b, rows, c) view into a NaN-filled (b, pre + rows + post, c + extra) buffer, holding data"""
    buf = torch.full((b, pre + rows + post, c + extra), NAN, device=DEV)
    v = buf[:, pre:pre + rows, :c]
    if data is not None:
        v.copy_(data)
    return v, buf


def outside(buf, v):
    """the bits of buf outside the view v (int32), to check that nothing outside an output view is written"""
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    off = v.storage_offset()
    row0 = off // buf.stride(1)
    mask[:, row0:row0 + v.shape[1], off % buf.stride(1):off % buf.stride(1) + v.shape[2]] = False
    return buf.view(torch.int32)[mask].clone()


def values(fam, shape, gen):
    """activation values of a family (float32, CPU)"""
    x = torch.randn(*shape, generator=gen)
    if fam == "small":
        x *= 1e-3
    elif fam == "large":
        x *= 1e4
    elif fam == "decades":
        x *= torch.logspace(-3, 3, shape[-1])
    elif fam == "spike":
        i = int(torch.randint(x.numel(), (1,), generator=gen))
        x.view(-1)[i] = 2.0 ** 11 * float(x.abs().max()) * (1 if i % 2 else -1)
    elif fam == "zeros":
        x[torch.rand(*shape, generator=gen) < 0.5] = 0.0
    elif fam == "allzero":
        x.zero_()
    return x


def weights(fam, cout, cin_g, k, gen):
    w = torch.randn(cout, cin_g, k, k, generator=gen) / (cin_g * k * k) ** 0.5
    if fam == "wdecades":
        w *= 10.0 ** (torch.rand(w.shape, generator=gen) * 6 - 3)
    return w


def conv_refs(x64, w64, bias64, z64, s, groups, a_scale, w_scale):
    """(ref, S, T) of conv(x, w) + bias (+ z) in float64 NCHW"""
    k = w64.shape[-1]
    conv = lambda a, ww: F.conv2d(a, ww, None, s, k // 2, groups=groups)  # noqa: E731
    ref, S = conv(x64, w64), conv(x64.abs(), w64.abs())
    T = 2.0 ** -25 / a_scale * conv(torch.ones_like(x64), w64.abs()) + 2.0 ** -25 / w_scale * conv(x64.abs(), torch.ones_like(w64))
    if bias64 is not None:
        ref, S = ref + bias64.view(1, -1, 1, 1), S + bias64.abs().view(1, -1, 1, 1)
    if z64 is not None:
        ref, S = ref + z64, S + z64.abs()
    return ref, S, T


def act_ref(act, ref, S, T):
    if act == cabi.ACT_RELU:
        return ref.clamp_min(0), S, T
    if act == cabi.ACT_SILU:
        want = F.silu(ref)
        return want, 1.1 * S + 4 * want.abs(), 1.1 * T
    return ref, S, T


def run_forward(case, k, s, ch, gen, check_name="fwd"):
    """one forward case of the table; returns what the gradient tests reuse"""
    cin, cout, groups = ch
    (h, w), b = case["hw"], case["b"]
    ho, wo = conv_out(h, w, k, s)
    wt = weights(case["fam"], cout, cin // groups, k, gen).to(DEV)
    xv, xbuf = fenced(b, h * w, cin, values(case["fam"], (b, h * w, cin), gen).to(DEV))
    bias = (torch.randn(cout, generator=gen) * 0.5).to(DEV) if case["bias"] else None
    f_hi, f_lo, _, _, w_scale = cabi.conv2d_f16x3_split_weight(wt, groups, dgrad=False)
    a_scale = cabi.pow2_scale(xbuf, 12)
    yv, ybuf = fenced(b, ho * wo, cout, pre=2, post=3)
    zdata = torch.randn(b, ho * wo, cout, generator=gen).to(DEV)
    z = None
    if case["z"] == "sep":
        z, _ = fenced(b, ho * wo, cout, zdata, pre=1, post=1)
    elif case["z"] == "alias":
        yv.copy_(zdata)
        z = yv
    before = outside(ybuf, yv)
    got = cabi.conv2d_f16x3(xv, (h, w), a_scale, f_hi, f_lo, w_scale, bias, groups, k, s, case["act"], out=yv, z=z)
    assert got is yv
    assert torch.equal(outside(ybuf, yv), before)
    x64, w64 = nchw(xv.double(), (h, w)), wt.double()
    ref, S, T = conv_refs(x64, w64, bias.double() if bias is not None else None,
                          nchw(zdata.double(), (ho, wo)) if z is not None else None, s, groups, float(a_scale), float(w_scale))
    want, S, T = act_ref(case["act"], ref, S, T)
    check_bound(check_name, nchw(got, (ho, wo)), want, S, T, C_FWD)
    if case["fam"] == "allzero":
        assert float(a_scale) == 1.0
    return xv, xbuf, wt


# ==== GPU: forward ========================================================================================================
@gpu
@pytest.mark.parametrize("k,s,ch", TABLE, ids=TABLE_IDS)
def test_forward_case_table(k, s, ch):
    """every map of the entry, with its act / bias / z / value family, within c (2^-24 S + T) of float64 F.conv2d; nothing
    outside the output view written"""
    gen = torch.Generator().manual_seed(1000 * k + 100 * s + CHANNELS.index(ch))
    for case in conv_cases(k, s, ch):
        run_forward(case, k, s, ch, gen)


@gpu
@pytest.mark.parametrize("name", sorted(REAL))
def test_real_layer_shapes(name):
    """the 800x1333 bs = 2 layers, each once: forward (ReLU, bias), input gradient and weight gradient against float64"""
    k, s, cin, cout, groups, h, w = REAL[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    case = dict(hw=(h, w), b=2, act=cabi.ACT_RELU, bias=True, z="none", fam="normal")
    xv, xbuf, wt = run_forward(case, k, s, (cin, cout, groups), gen, "fwd_real")
    ho, wo = conv_out(h, w, k, s)
    dyv, dybuf = fenced(2, ho * wo, cout, torch.randn(2, ho * wo, cout, generator=gen).to(DEV))
    ds, xs = cabi.pow2_scale(dybuf, 12), cabi.pow2_scale(xbuf, 12)
    _, _, d_hi, d_lo, w_scale = cabi.conv2d_f16x3_split_weight(wt, groups)
    dxv, dxbuf = fenced(2, h * w, cin)
    before = outside(dxbuf, dxv)
    cabi.conv2d_f16x3_dgrad(dyv, (ho, wo), ds, d_hi, d_lo, w_scale, groups, k, s, (h, w), out=dxv)
    assert torch.equal(outside(dxbuf, dxv), before)
    want, S, T = dgrad_refs(dyv, wt, (h, w), s, groups, float(ds), float(w_scale))
    check_bound("dgrad_real", nchw(dxv, (h, w)), want, S, T, C_DGRAD)
    dw = cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), wt.shape, s)
    want, S, T = wgrad_refs(dyv, xv, wt.shape, (h, w), s, groups, float(ds), float(xs))
    check_bound("wgrad_real", dw, want, S, T, C_WGRAD)


# ==== GPU: input gradient =================================================================================================
def dgrad_refs(dyv, wt, hw, s, groups, dy_scale, w_scale):
    b, k = dyv.shape[0], wt.shape[-1]
    ho, wo = conv_out(*hw, k, s)
    dy64, w64 = nchw(dyv.double(), (ho, wo)), wt.double()
    size = (b, w64.shape[1] * groups, *hw)
    gi = lambda g, ww: torch.nn.grad.conv2d_input(size, ww, g, s, k // 2, groups=groups)  # noqa: E731
    want, S = gi(dy64, w64), gi(dy64.abs(), w64.abs())
    T = 2.0 ** -25 / dy_scale * gi(torch.ones_like(dy64), w64.abs()) + 2.0 ** -25 / w_scale * gi(dy64.abs(), torch.ones_like(w64))
    return want, S, T


def mask_source(b, rows, c, gen):
    m = torch.randn(b, rows, c, generator=gen)
    r = torch.rand(b, rows, c, generator=gen)
    m[r < 0.15] = 0.0
    m[(r >= 0.15) & (r < 0.3)] = -0.0
    m[(r >= 0.3) & (r < 0.4)] = NAN
    return m


@gpu
@pytest.mark.parametrize("k,s,ch", TABLE, ids=TABLE_IDS)
def test_dgrad_case_table(k, s, ch):
    """input gradient at every map of the entry (every parity at stride 2), z absent / separate / aliasing dx, and the ReLU
    mask m (0 and -0.0 zero the value, NaN lets it through); at stride 1 without z and m the bits of the forward kernel on
    the flipped weights"""
    cin, cout, groups = ch
    gen = torch.Generator().manual_seed(2000 * k + 200 * s + CHANNELS.index(ch))
    wt = weights("normal", cout, cin // groups, k, gen).to(DEV)
    _, _, d_hi, d_lo, w_scale = cabi.conv2d_f16x3_split_weight(wt, groups)
    for case in conv_cases(k, s, ch):
        (h, w), b, mode = case["hw"], case["b"], case["dmode"]
        ho, wo = conv_out(h, w, k, s)
        dyv, dybuf = fenced(b, ho * wo, cout, values(case["dfam"], (b, ho * wo, cout), gen).to(DEV), pre=1, post=4)
        ds = cabi.pow2_scale(dybuf, 12)
        dxv, dxbuf = fenced(b, h * w, cin, pre=4, post=1)
        zdata = torch.randn(b, h * w, cin, generator=gen).to(DEV)
        msrc = mask_source(b, h * w, cin, gen).to(DEV)
        kw = {}
        if mode in ("z", "z_m_alias", "z_alias"):
            if mode == "z":
                kw["z"], _ = fenced(b, h * w, cin, zdata, pre=2, post=2)
            else:
                dxv.copy_(zdata)
                kw["z"] = dxv
        if mode in ("m", "z_m_alias"):
            kw["m"], _ = fenced(b, h * w, cin, msrc, pre=1, post=2, extra=8)
        before = outside(dxbuf, dxv)
        got = cabi.conv2d_f16x3_dgrad(dyv, (ho, wo), ds, d_hi, d_lo, w_scale, groups, k, s, (h, w), out=dxv, **kw)
        assert got is dxv and torch.equal(outside(dxbuf, dxv), before)
        want, S, T = dgrad_refs(dyv, wt, (h, w), s, groups, float(ds), float(w_scale))
        if "z" in kw:
            z64 = nchw(zdata.double(), (h, w))
            want, S = want + z64, S + z64.abs()
        got = nchw(got, (h, w))
        if "m" in kw:
            m64 = nchw(msrc.double(), (h, w))
            want = torch.ops.aten.threshold_backward(want, m64, 0)
            dead = ~(m64 > 0) & ~m64.isnan()
            assert bool((got[dead] == 0).all())
            assert torch.equal(got[dead].view(torch.int32), torch.zeros_like(got[dead]).view(torch.int32))  # +0.0
            S, T = S.masked_fill(dead, 0), T.masked_fill(dead, 0)
        check_bound("dgrad", got, want, S, T, C_DGRAD)
        if s == 1 and not kw:
            fwd = cabi.conv2d_f16x3(dyv, (h, w), ds, d_hi, d_lo, w_scale, None, groups, k, 1, 0)
            assert torch.equal(fwd.view(torch.int32), got.flatten(2).transpose(1, 2).contiguous().view(torch.int32))


# ==== GPU: weight gradient ================================================================================================
def wgrad_refs(dyv, xv, wshape, hw, s, groups, dy_scale, x_scale):
    k = wshape[-1]
    ho, wo = conv_out(*hw, k, s)
    dy64, x64 = nchw(dyv.double(), (ho, wo)), nchw(xv.double(), hw)
    gw = lambda a, g: torch.nn.grad.conv2d_weight(a, wshape, g, s, k // 2, groups=groups)  # noqa: E731
    want, S = gw(x64, dy64), gw(x64.abs(), dy64.abs())
    T = 2.0 ** -25 / dy_scale * gw(x64.abs(), torch.ones_like(dy64)) + 2.0 ** -25 / x_scale * gw(torch.ones_like(x64), dy64.abs())
    return want, S, T


@gpu
@pytest.mark.parametrize("k,s,ch", TABLE, ids=TABLE_IDS)
def test_wgrad_case_table(k, s, ch):
    """weight gradient at every map of the entry against float64 autograd; the same bits on a repeat and with the operands
    at other offsets and pitches"""
    cin, cout, groups = ch
    gen = torch.Generator().manual_seed(3000 * k + 300 * s + CHANNELS.index(ch))
    shape = (cout, cin // groups, k, k)
    for case in conv_cases(k, s, ch):
        (h, w), b = case["hw"], case["b"]
        ho, wo = conv_out(h, w, k, s)
        xd = values(case["fam"] if case["fam"] != "wdecades" else "decades", (b, h * w, cin), gen).to(DEV)
        dyd = values(case["dfam"], (b, ho * wo, cout), gen).to(DEV)
        xv, xbuf = fenced(b, h * w, cin, xd)
        dyv, dybuf = fenced(b, ho * wo, cout, dyd, pre=5, post=1)
        xs, ds = cabi.pow2_scale(xbuf, 12), cabi.pow2_scale(dybuf, 12)
        dw = cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), shape, s)
        assert torch.equal(dw, cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), shape, s))
        xv2, _ = fenced(b, h * w, cin, xd, pre=0, post=7, extra=12)
        dyv2, _ = fenced(b, ho * wo, cout, dyd, pre=2, post=0, extra=0)
        assert torch.equal(dw, cabi.conv2d_f16x3_wgrad(dyv2, ds, xv2, xs, (h, w), shape, s))
        want, S, T = wgrad_refs(dyv, xv, shape, (h, w), s, groups, float(ds), float(xs))
        check_bound("wgrad", dw, want, S, T, C_WGRAD)


@gpu
@pytest.mark.parametrize("name", sorted(WGRAD_SPLITS))
def test_wgrad_splits(name):
    """one split, one k-block per split, a short last split: float64 bound, repeat bits, other offsets and pitches, and
    cout_scale = the unscaled result times the scale, rounded once"""
    k, s, cin, cout, groups, h, w, b = WGRAD_SPLITS[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)))
    ho, wo = conv_out(h, w, k, s)
    shape = (cout, cin // groups, k, k)
    xd, dyd = torch.randn(b, h * w, cin, generator=gen).to(DEV), torch.randn(b, ho * wo, cout, generator=gen).to(DEV)
    xv, xbuf = fenced(b, h * w, cin, xd)
    dyv, dybuf = fenced(b, ho * wo, cout, dyd)
    xs, ds = cabi.pow2_scale(xbuf, 12), cabi.pow2_scale(dybuf, 12)
    sc = (torch.rand(cout, generator=gen) * 3 + 0.01).to(DEV)
    plain = cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), shape, s)
    scaled = cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), shape, s, cout_scale=sc)
    assert torch.equal(scaled, plain * sc.view(-1, 1, 1, 1))
    assert torch.equal(plain, cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (h, w), shape, s))
    xv2, _ = fenced(b, h * w, cin, xd, pre=9, post=0, extra=8)
    dyv2, _ = fenced(b, ho * wo, cout, dyd, pre=0, post=3, extra=64)
    assert torch.equal(scaled, cabi.conv2d_f16x3_wgrad(dyv2, ds, xv2, xs, (h, w), shape, s, cout_scale=sc))
    want, S, T = wgrad_refs(dyv, xv, shape, (h, w), s, groups, float(ds), float(xs))
    check_bound("wgrad_splits", plain, want, S, T, C_WGRAD)
    sc64 = sc.double().view(-1, 1, 1, 1)
    check_bound("wgrad_splits", scaled, want * sc64, S * sc64 + scaled.double().abs() / C_WGRAD, T * sc64, C_WGRAD)


@gpu
@pytest.mark.parametrize("name", [n for n in sorted(WGRAD_SPLITS) if not n.startswith("one_split")])
def test_wgrad_split_order(name):
    """the splits are summed in split order: dY is 0 except at the first pixel of each split, 2^24 in split 0 and 1 in the
    others, and x is 1 on the map, so every split's partial is exact; the in-order fp32 sum of the partials (2^24 + 1 rounds
    back to 2^24) is restated bit for bit, and any other order, or other split boundaries, give another result"""
    k, s, cin, cout, groups, h, w, b = WGRAD_SPLITS[name]
    ho, wo = conv_out(h, w, k, s)
    m = b * ho * wo
    splits, per, _ = wgrad_splits(m, wgrad_tiles(cin, cout, groups, k))
    assert splits > 2
    firsts = [j * per * KCV for j in range(splits)]
    dy = torch.zeros(m, cout)
    dy[firsts[0]] = 2.0 ** 24
    dy[firsts[1:]] = 1.0
    xv, xbuf = fenced(b, h * w, cin, torch.ones(b, h * w, cin, device=DEV))
    dyv, dybuf = fenced(b, ho * wo, cout, dy.view(b, ho * wo, cout).to(DEV))
    dw = cabi.conv2d_f16x3_wgrad(dyv, cabi.pow2_scale(dybuf, 12), xv, cabi.pow2_scale(xbuf, 12), (h, w),
                                 (cout, cin // groups, k, k), s)
    want = np.zeros((k, k), np.float32)
    exact = np.zeros((k, k))
    for ky in range(k):
        for kx in range(k):
            acc = np.float32(0)
            for j, f in enumerate(firsts):
                pix = f % (ho * wo)
                iy, ix = (pix // wo) * s - k // 2 + ky, (pix % wo) * s - k // 2 + kx
                part = np.float32(2.0 ** 24 if j == 0 else 1.0) * np.float32(0 <= iy < h and 0 <= ix < w)
                acc = np.float32(acc + part)
                exact[ky, kx] += float(part)
            want[ky, kx] = acc
    assert (exact != want).any()  # the order is visible
    want = torch.from_numpy(want).expand(cout, cin // groups, k, k)
    assert torch.equal(dw.cpu(), want)


# ==== GPU: non-finite locality ============================================================================================
LOCALITY = [  # (k, s, Cin, Cout, groups, H, W, b)
    (3, 1, 256, 512, 4, 7, 9, 2), (3, 2, 256, 256, 4, 8, 7, 2), (3, 2, 128, 64, 1, 13, 21, 1), (1, 2, 512, 256, 4, 6, 5, 2),
    (1, 1, 64, 128, 1, 5, 13, 1), (3, 2, 64, 64, 1, 1, 7, 2), (3, 1, 64, 64, 1, 1, 1, 2),
]


@gpu
@pytest.mark.parametrize("case", LOCALITY, ids=[f"k{c[0]}s{c[1]}_{c[2]}-{c[3]}g{c[4]}_{c[5]}x{c[6]}" for c in LOCALITY])
def test_non_finite_locality(case):
    """a NaN, +inf or -inf at one (pixel, channel) of x turns non-finite exactly the forward outputs and weight-gradient
    entries of receptive_fields_x (its own group only); one in dY exactly the input-gradient and weight-gradient entries of
    receptive_fields_dy; every other entry keeps the clean run's bits"""
    k, s, cin, cout, groups, H, W, b = case
    shape = (b, H, W, cin, cout, groups, k, s)
    ho, wo = conv_out(H, W, k, s)
    gen = torch.Generator().manual_seed(sum(case))
    wt = weights("normal", cout, cin // groups, k, gen).to(DEV)
    f_hi, f_lo, d_hi, d_lo, w_scale = cabi.conv2d_f16x3_split_weight(wt, groups)
    xv, xbuf = fenced(b, H * W, cin, torch.randn(b, H * W, cin, generator=gen).to(DEV))
    dyv, dybuf = fenced(b, ho * wo, cout, torch.randn(b, ho * wo, cout, generator=gen).to(DEV))
    xs, ds = cabi.pow2_scale(xbuf, 12), cabi.pow2_scale(dybuf, 12)
    wshape = (cout, cin // groups, k, k)
    fwd0 = cabi.conv2d_f16x3(xv, (H, W), xs, f_hi, f_lo, w_scale, None, groups, k, s, 0)
    dx0 = cabi.conv2d_f16x3_dgrad(dyv, (ho, wo), ds, d_hi, d_lo, w_scale, groups, k, s, (H, W))
    dw0 = cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (H, W), wshape, s)

    def same_elsewhere(got, clean, field):
        assert torch.equal(~got.isfinite(), field)
        assert torch.equal(got[~field].view(torch.int32), clean[~field].view(torch.int32))

    for i, bad in enumerate((NAN, float("inf"), -float("inf"))):
        n, y, x = (i % b, (i * 5) % H, (i * 3 + 2) % W) if i else (b - 1, H - 1, W - 1)
        c = [0, cin - 1, cin // 2 + 1][i]
        fwd_f, wg_f = receptive_fields_x(shape, n, y, x, c)
        keep = xv[n, y * W + x, c].item()
        xv[n, y * W + x, c] = bad
        got = cabi.conv2d_f16x3(xv, (H, W), xs, f_hi, f_lo, w_scale, None, groups, k, s, 0)
        same_elsewhere(got.view(b, ho, wo, cout).cpu(), fwd0.view(b, ho, wo, cout).cpu(), fwd_f)
        same_elsewhere(cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (H, W), wshape, s).cpu(), dw0.cpu(), wg_f)
        xv[n, y * W + x, c] = keep
        n, oy, ox, co = i % b, (i * 2 + 1) % ho, (i * 7) % wo, [cout - 1, 0, cout // 2 + 3][i]
        dx_f, wg_f = receptive_fields_dy(shape, n, oy, ox, co)
        keep = dyv[n, oy * wo + ox, co].item()
        dyv[n, oy * wo + ox, co] = bad
        got = cabi.conv2d_f16x3_dgrad(dyv, (ho, wo), ds, d_hi, d_lo, w_scale, groups, k, s, (H, W))
        same_elsewhere(got.view(b, H, W, cin).cpu(), dx0.view(b, H, W, cin).cpu(), dx_f)
        same_elsewhere(cabi.conv2d_f16x3_wgrad(dyv, ds, xv, xs, (H, W), wshape, s).cpu(), dw0.cpu(), wg_f)
        dyv[n, oy * wo + ox, co] = keep


# ==== GPU: split_weight ===================================================================================================
@gpu
@pytest.mark.parametrize("groups,cin,cout", [(1, 128, 64), (1, 64, 192), (4, 256, 512), (4, 512, 256)])
@pytest.mark.parametrize("k", [1, 3])
def test_split_weight_both_layouts(groups, cin, cout, k):
    """both layouts of the one-pass split equal split_f16_pair_dev of the permuted / flipped weight, bit for bit"""
    gen = torch.Generator().manual_seed(groups * 100 + cin + cout + k)
    w = (torch.randn(cout, cin // groups, k, k, generator=gen) * 10.0 ** (torch.rand(cout, cin // groups, k, k, generator=gen) * 6 - 4)).to(DEV)
    f_hi, f_lo, d_hi, d_lo, scale = cabi.conv2d_f16x3_split_weight(w, groups)
    assert torch.equal(scale, cabi.pow2_scale(w.contiguous(), 14))
    for (hi, lo), ref in (((f_hi, f_lo), w.permute(0, 2, 3, 1)), ((d_hi, d_lo), dgrad_weight(w, groups))):
        r_hi, r_lo, _ = cabi.split_f16_pair_dev(ref.contiguous(), scale)
        assert torch.equal(hi.view(torch.int16), r_hi.view(torch.int16)) and torch.equal(lo.view(torch.int16), r_lo.view(torch.int16))
    f2_hi, f2_lo, none_hi, none_lo, _ = cabi.conv2d_f16x3_split_weight(w, groups, dgrad=False)
    assert none_hi is None and none_lo is None and torch.equal(f2_hi, f_hi) and torch.equal(f2_lo, f_lo)


# ==== GPU: context gate ===================================================================================================
def gate_ref(y, x, z, w_mask, b_mask, w1, w2):
    """float64 restatement and its bound S: softmax(y.w + b) . y -> W1 -> ReLU -> W2 -> sigmoid -> gate * y + x (+ z).  S
    carries the logits' rounding (u times sum |y_c w_c| + |b|, the largest over the image, moves every softmax weight
    relatively by twice that) through the context, the two matrix products, the sigmoid's slope 1/4 and the last FMA."""
    y, x = y.double(), x.double()
    w_mask, b_mask, w1, w2 = w_mask.double(), b_mask.double(), w1.double(), w2.double()
    logit = y @ w_mask + b_mask
    p = logit.softmax(1)
    ctx = torch.einsum("npc,np->nc", y, p)
    hid = F.relu(ctx @ w1.T)
    gate = torch.sigmoid(hid @ w2.T)
    want = gate[:, None] * y + x + (z.double() if z is not None else 0.0)
    lerr = (y.abs() @ w_mask.abs() + b_mask.abs()).amax(1, keepdim=True)  # (b, 1)
    s_ctx = torch.einsum("npc,np->nc", y.abs(), p) * (1 + 2 * lerr)
    s_hid = s_ctx @ w1.abs().T + (ctx.abs() @ w1.abs().T)
    s_s = s_hid @ w2.abs().T + hid @ w2.abs().T
    S = y.abs() * (s_s / 4 + gate)[:, None] + (gate[:, None] * y).abs() + x.abs() + (z.double().abs() if z is not None else 0.0)
    return want, S


def gate_inputs(hw, b, C, r, gen):
    """y, x, z and the weights, with logits spanning +-100 in blocks: some chunks' exp(l - m) sums underflow against the
    image maximum"""
    w_mask = torch.randn(C, generator=gen)
    w_mask[0] = 4.0
    b_mask = torch.randn(1, generator=gen)
    y = torch.randn(b, hw, C, generator=gen)
    chunk_off = torch.linspace(-100, 90, gate_chunks(hw)[0])[torch.randperm(gate_chunks(hw)[0], generator=gen)]
    target = chunk_off.repeat_interleave(GATE_CHUNK)[:hw].view(1, hw) + 10 * torch.rand(b, hw, generator=gen)
    rest = (y[..., 1:].double() @ w_mask[1:].double() + b_mask.double())
    y[..., 0] = ((target.double() - rest) / 4.0).float()
    w1, w2 = torch.randn(r, C, generator=gen) / C ** 0.5, torch.randn(C, r, generator=gen) / r ** 0.5
    return y, torch.randn(b, hw, C, generator=gen), torch.randn(b, hw, C, generator=gen), w_mask, b_mask, w1, w2


@gpu
@pytest.mark.parametrize("hw,b,r,use_z", GATE_CASES)
def test_context_gate(hw, b, r, use_z):
    """float64 bound, repeat bits, nothing outside the output view written; a NaN in one pixel of image 0 turns all of image
    0 NaN, as torch's softmax does, and leaves the other images' bits unchanged"""
    C = 256
    gen = torch.Generator().manual_seed(hw * 10 + b + r)
    y, x, z, w_mask, b_mask, w1, w2 = gate_inputs(hw, b, C, r, gen)
    yv, _ = fenced(b, hw, C, y.to(DEV))
    xv, _ = fenced(b, hw, C, x.to(DEV), pre=1, post=0)
    zv = fenced(b, hw, C, z.to(DEV), pre=0, post=1)[0] if use_z else None
    ov, obuf = fenced(b, hw, C, pre=2, post=2)
    args = [t.to(DEV) for t in (w_mask, b_mask, w1, w2)]
    before = outside(obuf, ov)
    got = cabi.context_gate(yv, xv, *args, z=zv, out=ov)
    assert torch.equal(outside(obuf, ov), before)
    assert torch.equal(got.clone(), cabi.context_gate(yv, xv, *args, z=zv))
    if hw > GATE_CHUNK:  # some chunk's weights underflow against the image maximum
        logit = y.double() @ w_mask.double() + b_mask.double()
        assert float((logit.max(1).values - logit.min(1).values).min()) > 150
    want, S = gate_ref(y.to(DEV), x.to(DEV), z.to(DEV) if use_z else None, *[t.to(DEV) for t in (w_mask, b_mask, w1, w2)])
    check_bound("gate", got, want, S, torch.zeros_like(S), C_GATE)
    if b > 1:
        clean = got.clone()
        yv[0, hw // 2, 5] = NAN
        bad = cabi.context_gate(yv, xv, *args, z=zv)
        assert bool(bad[0].isnan().all())
        assert torch.equal(bad[1:].view(torch.int32), clean[1:].view(torch.int32))


# ==== GPU: upsample concat ================================================================================================
def ups_backward_f32(g, src, dst):
    """float32 restatement of the backward: each source sums its destination range, rows first, then columns, in order"""
    fy, fx = nearest_first_dst(src[0], dst[0]), nearest_first_dst(src[1], dst[1])
    b, _, C = g.shape
    gm = g.view(b, dst[0], dst[1], C)
    out = torch.zeros(b, src[0], src[1], C, device=g.device)
    ry, rx = int(np.diff(fy).max()), int(np.diff(fx).max())
    y0, x0 = torch.from_numpy(fy[:-1]).to(g.device), torch.from_numpy(fx[:-1]).to(g.device)
    ny, nx = torch.from_numpy(np.diff(fy)).to(g.device), torch.from_numpy(np.diff(fx)).to(g.device)
    for i in range(ry):
        for j in range(rx):
            ok = (i < ny)[:, None] & (j < nx)[None, :]
            iy, ix = (y0 + i).clamp_max(dst[0] - 1), (x0 + j).clamp_max(dst[1] - 1)
            v = gm[:, iy][:, :, ix]
            out = torch.where(ok[None, :, :, None], out + v, out)
    return out.view(b, src[0] * src[1], C)


@gpu
@pytest.mark.parametrize("src,dst", UPS_CASES)
def test_upsample_concat_and_backward(src, dst):
    """forward = [F.interpolate(nearest) | lo] bit for bit; backward = the float32 rows-then-columns restatement bit for
    bit, within c 2^-24 sum|g| of float64 autograd, and exactly 0 for sources no destination reads"""
    gen = torch.Generator().manual_seed(src[0] * 100 + dst[1])
    b, C = 2, 256
    hi, _ = fenced(b, src[0] * src[1], C, torch.randn(b, src[0] * src[1], C, generator=gen).to(DEV))
    lo, _ = fenced(b, dst[0] * dst[1], C, torch.randn(b, dst[0] * dst[1], C, generator=gen).to(DEV), pre=1, post=5)
    ov, obuf = fenced(b, dst[0] * dst[1], 2 * C)
    before = outside(obuf, ov)
    got = cabi.upsample_nearest_concat(hi, src, lo, dst, out=ov)
    assert torch.equal(outside(obuf, ov), before)
    up = tok(F.interpolate(nchw(hi, src), size=dst, mode="nearest"))
    assert torch.equal(got.view(torch.int32), torch.cat([up, lo], 2).view(torch.int32))
    gv, _ = fenced(b, dst[0] * dst[1], 2 * C, torch.randn(b, dst[0] * dst[1], 2 * C, generator=gen).to(DEV))
    g_hi = gv[:, :, :C]
    d = cabi.upsample_nearest_concat_backward(g_hi, dst, src)
    assert torch.equal(d.view(torch.int32), ups_backward_f32(g_hi, src, dst).view(torch.int32))
    h64 = nchw(hi.double(), src).requires_grad_(True)
    g64 = nchw(g_hi.double(), dst)
    (want,) = torch.autograd.grad(F.interpolate(h64, size=dst, mode="nearest"), h64, g64)
    (S,) = torch.autograd.grad(F.interpolate(h64, size=dst, mode="nearest"), h64, g64.abs())
    check_bound("upsample_bwd", nchw(d, src), want, S, torch.zeros_like(S), C_UPS)
    empty = torch.from_numpy(np.diff(nearest_first_dst(src[0], dst[0])) == 0)
    if bool(empty.any()):
        dm = d.view(b, src[0], src[1], C)[:, empty.to(DEV)]
        assert torch.equal(dm.view(torch.int32), torch.zeros_like(dm).view(torch.int32))


# ==== GPU: ResNet front end ===============================================================================================
@gpu
@pytest.mark.parametrize("b,H,W", [(2, 1, 1), (1, 1, 9), (2, 7, 1), (1, 33, 47), (2, 800, 1333)])
def test_stem_and_maxpool(b, H, W):
    """stem within c 2^-24 (|x| conv |w| + |bias|) of float64 (fp32 FMAs over 147 taps), then the maxpool on its output equal
    to torch's max_pool2d bit for bit"""
    gen = torch.Generator().manual_seed(b * 7 + H + W)
    x = torch.randn(b, 3, H, W, generator=gen).to(DEV)
    w = (torch.randn(64, 3, 7, 7, generator=gen) / 147 ** 0.5).to(DEV)
    bias = (torch.randn(64, generator=gen) * 0.1).to(DEV)
    wt = w.permute(1, 2, 3, 0).reshape(147, 64).contiguous()
    y = cabi.resnet_stem(x, wt, bias)
    ho, wo = conv_out(H, W, 7, 2)
    x64, w64 = x.double(), w.double()
    ref = F.relu(F.conv2d(x64, w64, bias.double(), 2, 3))
    S = F.conv2d(x64.abs(), w64.abs(), bias.double().abs(), 2, 3)
    check_bound("stem", nchw(y, (ho, wo)), ref, S, torch.zeros_like(S), C_STEM)
    p = cabi.maxpool3x3s2_tokens(y, (ho, wo))
    want = tok(F.max_pool2d(nchw(y, (ho, wo)), 3, 2, 1))
    assert torch.equal(p.view(torch.int32), want.contiguous().view(torch.int32))


@gpu
@pytest.mark.parametrize("b,H,W,C", [(2, 5, 7, 64), (1, 1, 1, 8), (2, 2, 9, 12), (1, 400, 667, 64)])
def test_maxpool_nan_signed_zero_and_negative_borders(b, H, W, C):
    """bit for bit with torch's max_pool2d on fp32: a NaN inside a window, all-negative windows at the padded border, and
    windows whose maximum is a tie of +0.0 and -0.0 in either order"""
    gen = torch.Generator().manual_seed(H * W + C)
    x = -torch.rand(b, C, H, W, generator=gen) - 0.5  # all negative: the padding must not win
    r = torch.rand(b, C, H, W, generator=gen)
    x[r < 0.2] = 0.0
    x[(r >= 0.2) & (r < 0.4)] = -0.0
    x[(r >= 0.4) & (r < 0.42)] = NAN
    x[:, :, 0, 0] = torch.tensor([0.0, -0.0, NAN, -3.0]).repeat(C)[:C]
    xv, _ = fenced(b, H * W, C, tok(x).to(DEV))
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    ov, obuf = fenced(b, ho * wo, C, pre=1, post=1)
    before = outside(obuf, ov)
    got = cabi.maxpool3x3s2_tokens(xv, (H, W), out=ov)
    assert torch.equal(outside(obuf, ov), before)
    want = tok(F.max_pool2d(x.to(DEV), 3, 2, 1)).contiguous()
    assert torch.equal(got.contiguous().view(torch.int32), want.view(torch.int32))
    assert bool((x.view(torch.int32) == 0).any()) and bool((x.view(torch.int32) == -2 ** 31).any()) and bool(x.isnan().any())


@gpu
def test_frozen_bn_fold_near_zero_variance():
    """w * s, s and bias - mean * s with s = weight * rsqrt(var + eps): var + eps near 0 (down to 2.5e-14, and 1e-30 with eps
    0), against float64 rounded once to fp32: within one rounding of it"""
    gen = torch.Generator().manual_seed(5)
    cout = 64
    w = torch.randn(cout, 32, 3, 3, generator=gen)
    var = torch.rand(cout, generator=gen)
    for eps, var_vals in ((1e-5, [-1e-5, -0.99999e-5, 0.0, 1e-12]), (0.0, [1e-30, 1e-38, 3e-20, 1.0])):
        var[:4] = torch.tensor(var_vals)
        bn = types.SimpleNamespace(weight=torch.randn(cout, generator=gen).to(DEV), bias=torch.randn(cout, generator=gen).to(DEV),
                                   running_mean=torch.randn(cout, generator=gen).to(DEV), running_var=var.clone().to(DEV), eps=eps)
        wf, s, bf = cabi.frozen_bn_fold(w.to(DEV), bn)
        s64 = bn.weight.double().cpu() * (bn.running_var.double().cpu() + eps).rsqrt()
        assert float(s64.abs().max()) > 1e5
        for got, ref in ((wf, w.double() * s64.view(-1, 1, 1, 1)), (s, s64), (bf, bn.bias.double().cpu() - bn.running_mean.double().cpu() * s64)):
            got = got.double().cpu()
            assert bool((got - ref).abs().le((1 + 2.0 ** -20) * U * ref.abs()).all())
