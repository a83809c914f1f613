"""FocalNetBackbone (focalnet.py): the reference's structure, initialisation, freezing and outputs on the CPU (fixture
tests/golden/focalnet_l_backbone.npz, made by tools/make_focalnet_golden.py from the reference itself), and on the H100 the token
path's kernels and the module against float64."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import salience_detr_b200 as pkg
from salience_detr_b200 import focalnet as fnm
from salience_detr_b200 import synthetic
from tools import make_focalnet_golden as mfg
from backbone_harness import (DEV, chain_graph_matches_eager,
                              check_no_sync_graph_replay_repeatability_and_launches, check_weight_loading, errors, golden,
                              mapper_chain, padded_images, rel_err, tf32)

FNB = pkg.FocalNetBackbone
TOKEN_ARCHS = ("focalnet_large_lrf", "focalnet_large_lrf_fl4")
FL4 = "focalnet_large_lrf_fl4"
U = 2.0 ** -24  # fp32 unit roundoff
_WEIGHTS = {}


def focalnet_weights(arch=FL4):
    """the fixture's synthetic weights for every key of ``arch``'s bare FocalNet"""
    if arch not in _WEIGHTS:
        net = fnm.FocalNet(**FNB._config(arch, {}))
        _WEIGHTS[arch] = synthetic.focalnet_weights(net.state_dict(), mfg.WEIGHT_SEED)
    return _WEIGHTS[arch]


def _backbone(arch=FL4, return_indices=(1, 2, 3), freeze_indices=(0,), **kw):
    return FNB(arch, weights=focalnet_weights(arch), return_indices=return_indices, freeze_indices=freeze_indices, **kw).eval()


# ---- CPU: the module against the reference --------------------------------------------------------------------------------
def test_state_dict_init_and_freeze_match_reference():
    g = golden("focalnet_l_backbone")
    m = _backbone()
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["shapes_json"]
    assert len(g["shapes_json"]) == 502 and [k for k in g["shapes_json"] if k.startswith("1.")] == [
        "1.norm1.weight", "1.norm1.bias", "1.norm2.weight", "1.norm2.bias", "1.norm3.weight", "1.norm3.bias"]
    assert {k: p.requires_grad for k, p in m.named_parameters()} == g["grad_json"]
    assert sum(g["grad_json"].values()) == 454
    assert m.num_channels == g["num_channels_json"] == [384, 768, 1536]
    m = FNB(FL4, return_indices=(1, 2, 3), freeze_indices=(0,))
    assert not m[0].patch_embed.training and not m[0].layers[0].training and m[0].layers[1].training
    assert all(float(v.sum()) == v.numel() * (1.0 if k.endswith("weight") else 0.0) for k, v in m[1].state_dict().items())
    torch.manual_seed(0)
    init = fnm.FocalNet(**FNB._config(FL4, {}))
    got = {k: float(v.double().sum()) for k, v in init.state_dict().items()}
    assert got.keys() == g["init_sums_json"].keys()
    assert all(got[k] == v for k, v in g["init_sums_json"].items())


def test_torch_forward_matches_reference():
    g = golden("focalnet_l_backbone")
    m = _backbone()
    with torch.no_grad():
        outs = m(g["image"])
    assert list(outs) == ["layers.1.blocks", "layers.2.blocks", "layers.3.blocks"]
    for k, v in outs.items():
        want = g[f"out.{k}"]
        assert v.shape == want.shape and v.is_contiguous()
        assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max()), k
    assert [tuple(v.shape[2:]) for v in outs.values()] == [(8, 13), (4, 7), (2, 4)]  # 61 x 99 -> 16 x 25 -> ...


@pytest.mark.parametrize("arch", sorted(FNB.model_arch))
def test_every_arch_builds(arch):
    m = FNB(arch)
    cfg = FNB.model_arch[arch]
    assert m.num_channels == [cfg["embed_dim"] * 2 ** i for i in range(4)]
    assert [len(m[0].layers[i].blocks) for i in range(4)] == list(cfg["depths"])
    assert not hasattr(m[0].layers[3], "downsample") and all(hasattr(m[0].layers[i], "downsample") for i in range(3))
    blocks = [blk for i in range(4) for blk in m[0].layers[i].blocks]
    assert blocks[0].drop_path.p == 0 and blocks[-1].drop_path.p == pytest.approx(cfg["stochastic_depth_prob"])
    ks = [fl[0].kernel_size[0] for fl in blocks[0].modulation.focal_layers]
    assert ks == [cfg["focal_windows"][0] + 2 * i for i in range(cfg["focal_levels"][0])]
    with torch.no_grad():
        outs = m(torch.randn(1, 3, 61, 94))
    assert [tuple(v.shape) for v in outs.values()] == [(1, c, math.ceil(16 / 2 ** i), math.ceil(24 / 2 ** i))
                                                       for i, c in enumerate(m.num_channels)]
    assert m.layers_supported() == (arch in TOKEN_ARCHS)


def test_return_indices_and_extractor_truncation():
    m = FNB("focalnet_tiny_srf", return_indices=(0, 1, 2))
    keys = list(m.state_dict())
    assert not any(k.startswith(("0.layers.3", "0.layers.2.downsample")) for k in keys)
    assert any(k.startswith("0.layers.1.downsample") for k in keys)
    assert [k for k in keys if k.startswith("1.")] == [f"1.norm{i}.{p}" for i in range(3) for p in ("weight", "bias")]
    m = FNB("focalnet_tiny_srf", return_indices=(2, 0))
    assert m.num_channels == [384, 96] and len(m[0].layers) == 3
    assert [k for k in m.state_dict() if k.startswith("1.")] == ["1.norm2.weight", "1.norm2.bias", "1.norm0.weight", "1.norm0.bias"]
    with torch.no_grad():
        assert list(m(torch.randn(1, 3, 32, 32))) == ["layers.2.blocks", "layers.0.blocks"]
    m = _backbone("focalnet_large_lrf", return_indices=(0,))
    assert len(m[0].layers) == 1 and not hasattr(m[0].layers[0], "downsample")
    assert m.launches_per_forward() == 1 + 2 * (14 + 3) + 1
    assert _backbone().launches_per_forward() == 445


def test_kwargs_work_as_in_reference():
    m = FNB("focalnet_tiny_srf", stochastic_depth_prob=0.1, mlp_ratio=2.0, return_indices=(0, 1, 2, 3))
    assert m[0].layers[3].blocks[-1].drop_path.p == pytest.approx(0.1) and m[0].layers[0].blocks[0].mlp.fc1.out_features == 192
    m = FNB("focalnet_tiny_srf", focal_levels=None, return_indices=(0,))  # None keeps the arch's value, as in the reference
    assert len(m[0].layers[0].blocks[0].modulation.focal_layers) == 2
    m = FNB(FL4, focal_levels=(2, 2, 2, 2), normalize_modulator=False, return_indices=(0,))
    mod = m[0].layers[0].blocks[0].modulation
    assert mod.focal_level == 2 and not mod.normalize_modulator and m.layers_supported()
    m = FNB(FL4, use_layerscale=False, return_indices=(0,))  # False is not None: it overrides the arch's True
    assert m[0].layers[0].blocks[0].gamma_1 == 1.0 and not m.layers_supported()
    m = FNB(FL4, dropout=0.1, return_indices=(0,))
    assert m[0].pos_drop.p == 0.1 and m[0].layers[0].blocks[0].mlp.drop.p == 0.1
    assert FNB._config("focalnet_tiny_srf", {})["use_conv_embed"] is False  # FocalNet's default fills what the arch leaves out
    with pytest.raises(TypeError, match="unexpected keyword"):
        FNB("focalnet_tiny_srf", layer_scale=0.5)


def test_weights_from_dict_model_and_path(tmp_path):
    # the weights are the bare FocalNet's, so the checks look at the feature extractor (backbone[0])
    check_weight_loading(tmp_path, lambda *a, **k: FNB(*a, **k)[0], "focalnet_tiny_srf", focalnet_weights, {},
                         classifier={"norm.weight": torch.ones(768), "norm.bias": torch.zeros(768),
                                     "head.weight": torch.zeros(1000, 768), "head.bias": torch.zeros(1000)},
                         drop="layers.0.blocks.0.modulation.h.bias", resize="patch_embed.proj.bias",
                         url="https://github.com/microsoft/FocalNet/releases/download/v1.0.0/focalnet_tiny_srf.pth",
                         bad_arch="focalnet_gigantic")


def test_tokens_supported_false_cases():
    m = FNB(FL4, freeze_indices=(0, 1, 2, 3))
    assert m.layers_supported()
    assert not m.tokens_supported(torch.randn(1, 3, 64, 64))  # CPU input
    for arch in ("focalnet_tiny_srf", "focalnet_base_lrf", "focalnet_xlarge_lrf", "focalnet_huge_fl4"):
        assert not FNB(arch).layers_supported(), arch
    m = FNB(FL4, return_indices=(0,))
    m[0].layers[0].blocks[1].mlp.act = nn.GELU(approximate="tanh")
    assert not m.layers_supported()
    m = FNB(FL4, focal_windows=(11, 11, 11, 11), focal_levels=(1, 1, 1, 1), return_indices=(0,))  # an 11 x 11 level
    assert not m.layers_supported()


# ---- GPU: kernels ---------------------------------------------------------------------------------------------------------
def _gelu64(x):
    return F.gelu(x)


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W", [(1, 1, 1), (2, 3, 5), (2, 61, 99), (2, 800, 1333)])
def test_focalnet_stem_vs_fp64(b, H, W):
    gen = torch.Generator().manual_seed(H * 13 + W)
    C = 192
    x = torch.randn(b, 3, H, W, generator=gen)
    w = torch.randn(C, 3, 7, 7, generator=gen) / 147 ** 0.5
    bias = torch.randn(C, generator=gen) * 0.1
    lg, lb = 1 + (torch.rand(C, generator=gen) - 0.5) * 0.5, torch.randn(C, generator=gen) * 0.1
    got = pkg.cabi.focalnet_stem(x.to(DEV), w.reshape(C, 147).t().contiguous().to(DEV), bias.to(DEV), lg.to(DEV),
                                 lb.to(DEV)).double()
    ho, wo = (H + 3) // 4, (W + 3) // 4
    assert tuple(got.shape) == (b, ho * wo, C)
    xd = F.pad(x.double().to(DEV), (0, 4 * wo - W, 0, 4 * ho - H))  # the reference's pad to a multiple of 4
    conv = F.conv2d(xd, w.double().to(DEV), bias.double().to(DEV), stride=4, padding=2).permute(0, 2, 3, 1).reshape(b, -1, C)
    ref = F.layer_norm(conv, (C,), lg.double().to(DEV), lb.double().to(DEV), 1e-5)
    s = F.conv2d(xd.abs(), w.double().to(DEV).abs(), bias.double().to(DEV).abs(), stride=4, padding=2)
    s = s.permute(0, 2, 3, 1).reshape(b, -1, C).amax(-1)
    # 147 products summed in fp32: |error| <= 150 u S before the LayerNorm, which divides by the row's std
    bound = 1e-5 + 160 * U * s / conv.std(-1, correction=0) * float(lg.abs().max())
    err = (got - ref).abs().amax(-1)
    assert bool((err <= bound).all()), float((err / bound).max())


FOCAL_MAPS = [(192, 2, (200, 336)), (192, 3, (9, 1)), (384, 2, (1, 1)), (384, 2, (25, 42)), (768, 1, (1, 37)),
              (768, 2, (13, 7)), (1536, 2, (4, 7)), (1536, 1, (2, 4))]


def _focal_inputs(C, b, hw, k, gen, ld=None):
    """fp32 ctx and gate as column slices of an f-like output (b, n, ld), a depthwise weight, and a prior ctx_all"""
    n = hw[0] * hw[1]
    ld = ld or 2 * C + 8
    fo = torch.randn(b, n, ld, generator=gen)
    w = torch.randn(C, 1, k, k, generator=gen) / k
    prior = torch.randn(b, n, C, generator=gen)
    return fo.to(DEV), w.to(DEV), prior.to(DEV)


def _level_ref(ctx, w, hw):
    """GELU(dwconv(ctx)) in float64 and the bound S = dwconv(|ctx|, |w|) of its fp32 error: (b, n, C) each"""
    b, n, C = ctx.shape
    k = w.shape[-1]
    x = ctx.double().reshape(b, hw[0], hw[1], C).permute(0, 3, 1, 2)
    conv = F.conv2d(x, w.double(), padding=k // 2, groups=C)
    s = F.conv2d(x.abs(), w.double().abs(), padding=k // 2, groups=C)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(b, n, C)  # noqa: E731
    p = _gelu64(flat(conv))
    # k^2 fp32 FMAs (|error| <= k^2 u S), GELU's slope below 1.13, erff and its products a few ulps of p
    return p, 1.13 * k * k * U * flat(s) + 8 * U * p.abs() + 1e-37


@pytest.mark.gpu
@pytest.mark.parametrize("k", [3, 5, 7, 9])
@pytest.mark.parametrize("case", range(len(FOCAL_MAPS)))
def test_focal_level_vs_fp64(case, k):
    C, b, hw = FOCAL_MAPS[case]
    gen = torch.Generator().manual_seed(case * 10 + k)
    fo, w, prior = _focal_inputs(C, b, hw, k, gen)
    ctx, gate = fo[..., C:2 * C], fo[..., 2 * C + 1:2 * C + 2]
    wk = w.reshape(C, k * k).t().contiguous()
    p_ref, p_bound = _level_ref(ctx, w, hw)
    g = gate.double()
    for first in (True, False):
        ctx_all = prior.clone()
        p = pkg.cabi.focal_level_tokens(ctx, gate, hw, wk, ctx_all, first)
        err = (p.double() - p_ref).abs()
        assert bool((err <= p_bound).all()), float((err / p_bound).max())
        before = 0 if first else prior.double()
        ref = before + p_ref * g
        bound = g.abs() * p_bound + 2 * U * (before.abs() if not first else 0) + 2 * U * (p_ref * g).abs() + 1e-37
        assert bool(((ctx_all.double() - ref).abs() <= bound).all())
        # the product and the sum are rounded on their own, as in torch: the same bits from the kernel's own p
        want = (0 + p * gate) if first else prior + p * gate
        assert torch.equal(ctx_all, want)
    # the last level: no ctx written, the same ctx_all
    ctx_all2 = prior.clone()
    parts = pkg.cabi.focal_context_partials(b, hw, C, fo.device)
    assert pkg.cabi.focal_level_tokens(ctx, gate, hw, wk, ctx_all2, False, out=False, partials=parts) is None
    assert torch.equal(ctx_all2, ctx_all)


def _tiles(hw):
    n = hw[0] * hw[1]
    r = max(1, -(-n // 1024))
    return r, -(-n // (8 * r))


@pytest.mark.gpu
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("C,b,hw", [(192, 2, (200, 336)), (384, 2, (1, 1)), (768, 2, (1, 37)), (1536, 3, (13, 7)),
                                    (192, 1, (41, 29))])
def test_global_context_vs_fp64_and_repeatable(C, b, hw, normalize):
    k, L = 9, 4
    gen = torch.Generator().manual_seed(C + hw[0] + normalize)
    fo, w, prior = _focal_inputs(C, b, hw, k, gen)
    ctx, gate_l, gate_g = fo[..., C:2 * C], fo[..., 2 * C + 3:2 * C + 4], fo[..., 2 * C + 4:2 * C + 5]
    wk = w.reshape(C, k * k).t().contiguous()
    parts = pkg.cabi.focal_context_partials(b, hw, C, fo.device)
    ctx_all = prior.clone()
    pkg.cabi.focal_level_tokens(ctx, gate_l, hw, wk, ctx_all, False, out=False, partials=parts)
    before = ctx_all.double()
    out = pkg.cabi.focal_global_context(parts, gate_g, hw, ctx_all.clone(), L, normalize)
    again = pkg.cabi.focal_global_context(parts, gate_g, hw, ctx_all.clone(), L, normalize)
    assert torch.equal(out, again)
    p_ref, p_bound = _level_ref(ctx, w, hw)
    n = hw[0] * hw[1]
    r, tiles = _tiles(hw)
    mean = p_ref.mean(1, keepdim=True)
    # the fixed-order sum: R terms per warp, 8 warps, tiles / 8 + 1 per reduction warp, 8 more
    mean_bound = p_bound.mean(1, keepdim=True) + (r + tiles // 8 + 18) * U * p_ref.abs().mean(1, keepdim=True)
    m = _gelu64(mean)
    g = gate_g.double()
    ref = before + m * g
    bound = 1.13 * mean_bound * g.abs() + 8 * U * (m * g).abs() + 2 * U * (before.abs() + (m * g).abs())
    if normalize:
        ref, bound = ref / (L + 1), bound / (L + 1) + U * (ref / (L + 1)).abs()
    err = (out.double() - ref).abs()
    assert bool((err <= bound + 1e-37).all()), float((err / (bound + 1e-37)).max())


@pytest.mark.gpu
def test_focal_context_nan_poisons_what_torch_poisons():
    """a NaN pixel of the context poisons its k x k neighbourhoods level by level and, through the global mean, its whole image,
    and nothing in the other image"""
    C, b, hw, L = 192, 2, (13, 21), 3
    gen = torch.Generator().manual_seed(5)
    fo, _, _ = _focal_inputs(C, b, hw, 3, gen)
    fo[1, 4 * hw[1] + 6, C + 7] = float("nan")
    ks = [3, 5, 7]
    ws = [(torch.randn(C, 1, kk, kk, generator=gen) / kk).to(DEV) for kk in ks]
    ctx_all = torch.empty(b, hw[0] * hw[1], C, device=DEV)
    parts = pkg.cabi.focal_context_partials(b, hw, C, DEV)
    ctx, seen = fo[..., C:2 * C], []
    for level, w in enumerate(ws):
        last = level + 1 == L
        wk = w.reshape(C, -1).t().contiguous()
        ctx = pkg.cabi.focal_level_tokens(ctx, fo[..., 2 * C + level:2 * C + level + 1], hw, wk, ctx_all, level == 0, out=True,
                                          partials=parts if last else None)
        seen.append(ctx.isnan())
    pkg.cabi.focal_global_context(parts, fo[..., 2 * C + L:2 * C + L + 1], hw, ctx_all, L, True)
    # the reference's chain in float64
    mod = fnm.FocalModulation(C, focal_level=L, focal_window=3, normalize_modulator=True).double().to(DEV)
    x = fo.double().reshape(b, hw[0], hw[1], -1).permute(0, 3, 1, 2)
    rctx, gates, rall = x[:, C:2 * C], x[:, 2 * C:], 0
    with torch.no_grad():
        for level, w in enumerate(ws):
            rctx = F.gelu(F.conv2d(rctx, w.double(), padding=ks[level] // 2, groups=C))
            assert torch.equal(seen[level], rctx.permute(0, 2, 3, 1).reshape(b, -1, C).isnan())
            rall = rall + rctx * gates[:, level:level + 1]
        rall = (rall + F.gelu(rctx.mean(2, keepdim=True).mean(3, keepdim=True)) * gates[:, L:L + 1]) / (L + 1)
    want = rall.permute(0, 2, 3, 1).reshape(b, -1, C)
    assert torch.equal(ctx_all.isnan(), want.isnan())
    # depthwise levels: the NaN stays in its channel, where the mean spreads it over the whole image
    assert bool(want[1, :, 7].isnan().all()) and int(want.isnan().sum()) == hw[0] * hw[1]
    del mod


@pytest.mark.gpu
@pytest.mark.parametrize("C,rows", [(192, 1), (384, 1000), (1536, 77), (768, 134400 // 4)])
def test_modulate_is_torch_product(C, rows):
    gen = torch.Generator().manual_seed(C + rows)
    fo = torch.randn(1, rows, 2 * C + 8, generator=gen).to(DEV)
    fo[0, 0, 3] = float("nan")
    h = torch.randn(1, rows, C, generator=gen).to(DEV)
    want = fo[..., :C] * h
    assert torch.equal(pkg.cabi.focal_modulate(fo[..., :C], h).isnan(), want.isnan())
    got = pkg.cabi.focal_modulate(fo[..., :C], h, out=h)
    assert got.data_ptr() == h.data_ptr() and torch.equal(got.nan_to_num(), want.nan_to_num())


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(1, 64), (333, 192), (1000, 384), (77, 768), (129, 1536), (134400, 192)])
def test_layernorm_scale_add_vs_fp64(rows, C):
    gen = torch.Generator().manual_seed(rows + C)
    y = torch.randn(rows, C, generator=gen) * 2 + 0.5
    y[0] = 1.25
    t = torch.randn(rows, C, generator=gen)
    if rows > 2:
        y[1, 7] = float("nan")
        y[2] = 1e4 + torch.randn(C, generator=gen) * 1e-2
    lg, lb = 1 + (torch.rand(C, generator=gen) - 0.5) * 0.5, torch.randn(C, generator=gen) * 0.1
    gamma = 0.05 + torch.rand(C, generator=gen)
    got = pkg.cabi.layernorm_scale_add_tokens_(t.clone().to(DEV), y.to(DEV), lg.to(DEV), lb.to(DEV), gamma.to(DEV)).cpu().double()
    ln = F.layer_norm(y.double(), (C,), lg.double(), lb.double(), 1e-5)
    ref = t.double() + gamma.double() * ln
    assert torch.equal(got.isnan(), ref.isnan())
    assert torch.allclose(got[0], t[0].double() + gamma.double() * lb.double(), atol=1e-6)
    yd = y.double()
    ln_bound = 1e-5 * (1 + yd.mean(1, keepdim=True).abs() / (yd.std(1, correction=0, keepdim=True) + 1e-3))
    bound = gamma.double() * ln_bound + 2 * U * (t.double().abs() + (gamma.double() * ln).abs())
    err = (got - ref).nan_to_num().abs()
    assert bool((err <= bound.nan_to_num()).all()), float((err / bound).nan_to_num().max())


# ---- GPU: forward_tokens --------------------------------------------------------------------------------------------------
FWD_CASES = {
    "fl4_64x100": (FL4, (1, 2, 3), 2, 64, 100),
    "fl4_ragged_all": (FL4, (0, 1, 2, 3), 3, 200, 312),
    "fl4_config2": (FL4, (1, 2, 3), 2, 800, 1344),
    "lrf_ragged": ("focalnet_large_lrf", (1, 2, 3), 2, 150, 230),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(FWD_CASES))
def test_forward_tokens_vs_fp64(case):
    """Every output within 16x the error of the same forward() in torch fp32 (TF32 off), measured here, and below a tenth of
    TF32's."""
    arch, ri, b, H, W = FWD_CASES[case]
    m = _backbone(arch, return_indices=ri).to(DEV)
    x = padded_images(b, H, W, torch.Generator().manual_seed(H + W)).to(DEV)
    with torch.no_grad():
        assert m.tokens_supported(x)
    errs, tok = errors(m, x)
    assert list(tok) == [f"layers.{i}.blocks" for i in ri]
    for k, (e_tok, e_fp32, e_tf32) in errs.items():
        print(f"{case} {k}: tokens {e_tok:.3e}  torch fp32 {e_fp32:.3e}  TF32 {e_tf32:.3e}")
        assert e_tok <= 16 * e_fp32 and e_tok < 0.1 * e_tf32, (k, e_tok, e_fp32, e_tf32)
    for k, v in tok.items():
        bb, c, h, w = v.shape
        assert v.stride() == (h * w * c, 1, w * c, c) and v.is_contiguous(memory_format=torch.channels_last)
        assert v._base is not None and v._base.shape == (bb, h * w, c)  # a view of its own token buffer
    ptrs = [v.data_ptr() for v in tok.values()]
    assert len(set(ptrs)) == len(ptrs)


@pytest.mark.gpu
def test_golden_outputs_on_gpu():
    """The token path on the fixture's image within 1e-5 of the largest output of the fixture's outputs, beyond their own distance
    from float64: the reference's fp32 CPU forward of these 24 post-LN blocks is itself about 1.2e-5 of the largest value away
    from float64 at layers.2, which leaves backbone_harness.check_golden_outputs_on_gpu's plain 1e-5 no room."""
    g = golden("focalnet_l_backbone")
    m = _backbone().to(DEV)
    x = g["image"].to(DEV)
    with torch.no_grad():
        assert m.tokens_supported(x)
        outs = m(x)
        ref = copy.deepcopy(m).double()(x.double())
    for k, v in outs.items():
        want = g[f"out.{k}"].to(DEV)
        own = float((want.double() - ref[k]).abs().max())
        print(f"{k}: tokens - fixture {float((v - want).abs().max()):.3e}, fixture - float64 {own:.3e}")
        assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max()) + own, k


@pytest.mark.gpu
def test_no_sync_graph_replay_repeatability_and_launches():
    m = _backbone().to(DEV)
    x = padded_images(2, 97, 131, torch.Generator().manual_seed(3)).to(DEV)
    check_no_sync_graph_replay_repeatability_and_launches(m, x, 445)


@pytest.mark.gpu
def test_kernel_weights_follow_parameter_changes():
    m = _backbone().to(DEV)
    x = padded_images(1, 64, 100, torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        outs = [m(x)["layers.3.blocks"].clone()]
        m[0].layers[2].blocks[3].gamma_1.mul_(0.5)
        outs.append(m(x)["layers.3.blocks"].clone())
        m[0].layers[1].blocks[1].modulation.focal_layers[2][0].weight.mul_(-1.0)
        outs.append(m(x)["layers.3.blocks"].clone())
        m[1].norm3.weight.mul_(1.5)
        outs.append(m(x)["layers.3.blocks"])
        want = copy.deepcopy(m).double()(x.double())["layers.3.blocks"]
    assert all(not torch.equal(a, b) for a, b in zip(outs, outs[1:]))
    assert rel_err(outs[-1], want) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["input_grad", "param_grad", "stochastic_depth", "focalnet_tiny_srf"])
def test_torch_path_on_cuda_is_the_op_chain(name):
    arch = name if name.startswith("focalnet_") else FL4
    m = FNB(arch, return_indices=(1, 2, 3), freeze_indices=(0, 1, 2, 3) if name != "param_grad" else (0,)).to(DEV).eval()
    x = padded_images(1, 64, 96, torch.Generator().manual_seed(5)).to(DEV)
    if name == "input_grad":
        x.requires_grad_(True)
    if name == "stochastic_depth":
        m.train()
    ctx = torch.enable_grad() if name in ("input_grad", "param_grad") else torch.no_grad()
    with ctx:
        assert not m.tokens_supported(x)
        if name == "stochastic_depth":
            m.eval()
            assert m.tokens_supported(x)
            return
        n0 = pkg.cabi.launch_count()
        got = m(x)
        assert pkg.cabi.launch_count() == n0
        want = m.forward_torch(x)
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in got)
    if name in ("input_grad", "param_grad"):
        with pytest.raises(RuntimeError, match="needs forward"):
            with torch.enable_grad():
                m.forward_tokens(x)


# ---- GPU: backbone -> ChannelMapper -> encoder ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_backbone_mapper_encoder_chain():
    """images -> FocalNet-L (channels-last views) -> ChannelMapper(in_channels=num_channels) with zero transposes ->
    forward_encoder: the mapper's tokens within 8x the error of the torch fp32 backbone chain against the float64 backbone, and
    the whole chain in one CUDA graph"""
    bb = _backbone().to(DEV)
    c = mapper_chain(bb)
    with torch.no_grad(), tf32(False):
        fp32_feats = bb.forward_torch(c.x)
    with torch.no_grad():
        fp32_mapped = c.mapper.forward_tokens({k: v.contiguous(memory_format=torch.channels_last)
                                               for k, v in fp32_feats.items()})[0]
    e_tok, e_fp32 = rel_err(c.mapped, c.ref_mapped.double()), rel_err(fp32_mapped, c.ref_mapped.double())
    print(f"mapper tokens: backbone tokens {e_tok:.3e}, torch fp32 {e_fp32:.3e}")
    assert e_tok <= 8 * e_fp32
    assert chain_graph_matches_eager(bb, c)
