"""ConvNeXtBackbone (convnext.py): the reference's structure, initialisation, freezing and outputs on the CPU (fixture
tests/golden/convnext_l_backbone.npz, made by tools/make_convnext_golden.py from the reference itself), and on the H100 the token
path's kernels, the extended projection GEMM and the module against float64."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import salience_detr_b200 as pkg
from salience_detr_b200 import convnext as cnm
from backbone_harness import (DEV, chain_graph_matches_eager, check_golden_outputs_on_gpu,
                              check_no_sync_graph_replay_repeatability_and_launches, check_weight_loading, convnext_weights,
                              errors, golden, mapper_chain, padded_images, rel_err, tf32)
from backbone_harness import convnext_backbone as _backbone

CNB = pkg.ConvNeXtBackbone


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_state_dict_init_and_freeze_match_reference():
    g = golden("convnext_l_backbone")
    m = _backbone()
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["shapes_json"]
    assert len(g["shapes_json"]) == 340 and not any(k.startswith("classifier.") for k in g["shapes_json"])
    assert {k: p.requires_grad for k, p in m.named_parameters()} == g["grad_json"]
    assert m.num_channels == g["num_channels_json"] == [384, 768, 1536]
    m = CNB("conv_l", return_indices=(1, 2, 3), freeze_indices=(0,))
    assert not m.features[0].training and not m.features[1].training and not m.features[2].training and m.features[3].training
    torch.manual_seed(0)
    init = CNB("conv_l")
    got = {k: float(v.double().sum()) for k, v in init.state_dict().items()}
    assert got.keys() == g["init_sums_json"].keys()
    assert all(got[k] == v for k, v in g["init_sums_json"].items())
    assert float(init.features[1][0].layer_scale.max()) == float(init.features[1][0].layer_scale.min()) == pytest.approx(1e-6)


def test_torch_forward_matches_reference():
    g = golden("convnext_l_backbone")
    m = _backbone()
    with torch.no_grad():
        outs = m(g["image"])
    assert list(outs) == ["features.3", "features.5", "features.7"]
    for k, v in outs.items():
        want = g[f"out.{k}"]
        assert v.shape == want.shape
        assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max()), k


@pytest.mark.parametrize("arch", sorted(CNB.model_arch))
def test_every_arch_builds(arch):
    m = CNB(arch)
    setting = CNB.model_arch[arch]["block_setting"]
    assert m.num_channels == [s.input_channels for s in setting]
    assert not hasattr(m, "classifier") and len(m.features) == 8
    blocks = [blk for i in range(4) for blk in m.features[2 * i + 1]]
    assert [len(m.features[2 * i + 1]) for i in range(4)] == [s.num_layers for s in setting]
    p = CNB.model_arch[arch]["stochastic_depth_prob"]
    assert blocks[0].stochastic_depth.p == 0 and blocks[-1].stochastic_depth.p == pytest.approx(p)
    with torch.no_grad():
        outs = m(torch.randn(1, 3, 64, 96))
    assert [tuple(v.shape) for v in outs.values()] == [(1, c, 16 // 2 ** i, 24 // 2 ** i) for i, c in enumerate(m.num_channels)]
    assert m.layers_supported() == (arch in ("conv_b", "conv_l"))


def test_return_indices_and_extractor_truncation():
    m = CNB("conv_b", return_indices=(2, 0))
    assert m.num_channels == [512, 128] and len(m.features) == 6
    assert not any(k.startswith(("features.6", "features.7")) for k in m.state_dict())
    with torch.no_grad():
        assert list(m(torch.randn(1, 3, 32, 32))) == ["features.5", "features.1"]
    m = CNB("conv_b", return_indices=(0,))
    assert len(m.features) == 2 and m.launches_per_forward() == 1 + 5 * 3


def test_kwargs_work_as_in_reference():
    m = CNB("conv_b", layer_scale=0.5, stochastic_depth_prob=0.2, return_indices=(0, 1, 2, 3))
    assert float(m.features[3][0].layer_scale.mean()) == 0.5
    assert m.features[7][-1].stochastic_depth.p == pytest.approx(0.2)
    m = CNB("conv_b", norm_layer=nn.Identity, return_indices=(0,))
    assert type(m.features[0][1]) is nn.Identity and not m.layers_supported()

    class MyBlock(cnm.CNBlock):
        pass

    m = CNB("conv_b", block=MyBlock, return_indices=(0,))
    assert type(m.features[1][0]) is MyBlock and not m.layers_supported()


def test_weights_from_dict_model_and_path(tmp_path):
    check_weight_loading(tmp_path, CNB, "conv_b", convnext_weights, {},
                         classifier={"classifier.0.weight": torch.ones(1024), "classifier.0.bias": torch.zeros(1024),
                                     "classifier.2.weight": torch.zeros(1000, 1024), "classifier.2.bias": torch.zeros(1000)},
                         drop="features.1.0.layer_scale", resize="features.0.0.bias",
                         url="https://download.pytorch.org/models/convnext_base-6075fbad.pth", bad_arch="conv_xl")


def test_tokens_supported_false_cases():
    m = CNB("conv_b", freeze_indices=(0, 1, 2, 3))
    assert m.layers_supported()
    assert not m.tokens_supported(torch.randn(1, 3, 64, 64))  # CPU input
    assert not CNB("conv_t").layers_supported() and not CNB("conv_s").layers_supported()  # 96-wide stages
    assert not CNB("conv_b", norm_layer=partial_ln()).layers_supported()
    m = CNB("conv_b", return_indices=(0,))
    m.features[1][0].block[4] = nn.GELU(approximate="tanh")
    assert not m.layers_supported()


def partial_ln():
    from functools import partial

    return partial(nn.GroupNorm, 1)


def test_space_to_depth_reproduces_the_2x2_convolution():
    """the downsample as one GEMM: rows (dy, dx, c) of the (H / 2) x (W / 2) map against the weight permuted to (Cout, 2, 2, Cin)
    equal F.conv2d(k=2, s=2) in float64, odd sizes dropping the last row / column"""
    g = torch.Generator().manual_seed(5)
    for b, c, cout, H, W in [(2, 8, 12, 7, 9), (1, 4, 6, 5, 4), (1, 3, 5, 2, 3), (2, 6, 4, 10, 1)]:
        x = torch.randn(b, c, H, W, generator=g, dtype=torch.float64)
        w = torch.randn(cout, c, 2, 2, generator=g, dtype=torch.float64)
        bias = torch.randn(cout, generator=g, dtype=torch.float64)
        ho, wo = H // 2, W // 2
        rows = x[:, :, :2 * ho, :2 * wo].reshape(b, c, ho, 2, wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(b, ho * wo, 4 * c)
        got = rows @ w.permute(0, 2, 3, 1).reshape(cout, 4 * c).t() + bias
        want = F.conv2d(x, w, bias, stride=2) if ho and wo else torch.zeros(b, cout, ho, wo, dtype=torch.float64)
        assert torch.allclose(got.view(b, ho, wo, cout).permute(0, 3, 1, 2), want, rtol=1e-12, atol=1e-12)


# ---- GPU: kernels -----------------------------------------------------------------------------------------------------
def _rows(x):
    b, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(b, h * w, c).contiguous()


def _maps(t, hw):
    b, _, c = t.shape
    return t.view(b, hw[0], hw[1], c).permute(0, 3, 1, 2)


def _ln64(x, g, b, eps=1e-6):
    """float64 LayerNorm over dim 1 of an NCHW map"""
    return F.layer_norm(x.permute(0, 2, 3, 1), x.shape[1:2], g.double(), b.double(), eps).permute(0, 3, 1, 2)


def _ln_affine(c, gen):
    return 1 + (torch.rand(c, generator=gen) - 0.5) * 0.5, torch.randn(c, generator=gen) * 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W,C", [(2, 64, 96, 192), (1, 7, 13, 128), (3, 5, 4, 192), (1, 4, 4, 1536), (2, 803, 1343, 192),
                                     (1, 3, 40, 128), (2, 40, 2, 192)])
def test_stem_vs_fp64(b, H, W, C):
    gen = torch.Generator().manual_seed(b * 1000 + H * 7 + W + C)
    x = torch.randn(b, 3, H, W, generator=gen) * 2
    w = torch.randn(C, 3, 4, 4, generator=gen) / 48 ** 0.5
    bias = torch.randn(C, generator=gen) * 0.1
    lg, lb = _ln_affine(C, gen)
    got = pkg.cabi.convnext_stem(x.to(DEV), w.reshape(C, 48).t().contiguous().to(DEV), bias.to(DEV), lg.to(DEV), lb.to(DEV))
    ho, wo = H // 4, W // 4
    assert tuple(got.shape) == (b, ho * wo, C)
    if ho == 0 or wo == 0:
        return
    ref = _ln64(F.conv2d(x.double(), w.double(), bias.double(), 4), lg, lb)
    err = float((_maps(got.cpu().double(), (ho, wo)) - ref).abs().max())
    assert err <= 2e-5 * float(ref.abs().max()), err


def _dw_case(b, H, W, C, gen, scale=1.0):
    x = torch.randn(b, C, H, W, generator=gen) * scale
    w = torch.randn(C, 1, 7, 7, generator=gen) / 7
    bias = torch.randn(C, generator=gen) * 0.1
    lg, lb = _ln_affine(C, gen)
    return x, w, bias, lg, lb


def _dwconv(x, w, bias, lg, lb):
    b, C, H, W = x.shape
    return pkg.cabi.dwconv7x7_layernorm_tokens(_rows(x).to(DEV), (H, W), w.reshape(C, 49).t().contiguous().to(DEV), bias.to(DEV),
                                               lg.to(DEV), lb.to(DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W", [(2, 1, 1), (1, 2, 3), (2, 7, 200), (1, 25, 42), (2, 50, 84), (1, 200, 336), (3, 9, 4)])
@pytest.mark.parametrize("C", [128, 192, 384, 768, 1536])
def test_dwconv_layernorm_vs_fp64(b, H, W, C):
    if H * W > 20000 and C > 384:
        pytest.skip("the largest maps run at the stage-1 widths they have in the backbone")
    gen = torch.Generator().manual_seed(H * 31 + W + C + b)
    x, w, bias, lg, lb = _dw_case(b, H, W, C, gen)
    xr = _rows(x).to(DEV)
    xc = xr.clone()
    got = pkg.cabi.dwconv7x7_layernorm_tokens(xr, (H, W), w.reshape(C, 49).t().contiguous().to(DEV), bias.to(DEV), lg.to(DEV),
                                              lb.to(DEV))
    assert torch.equal(xr, xc)  # the block input stays untouched
    ref = _ln64(F.conv2d(x.double(), w.double(), bias.double(), padding=3, groups=C), lg, lb)
    err = float((_maps(got.cpu().double(), (H, W)) - ref).abs().max())
    assert err <= 2e-5 * float(ref.abs().max()), err


@pytest.mark.gpu
def test_dwconv_layernorm_nan_and_constant_rows():
    gen = torch.Generator().manual_seed(9)
    b, H, W, C = 1, 20, 30, 192
    x, w, bias, lg, lb = _dw_case(b, H, W, C, gen)
    x[0, 5, 10, 12] = float("nan")
    got = _maps(_dwconv(x, w, bias, lg, lb).cpu(), (H, W))
    ref = _ln64(F.conv2d(x.double(), w.double(), bias.double(), padding=3, groups=C), lg, lb)
    nan_tok = ref.isnan().any(1)
    assert int(nan_tok.sum()) == 49 and torch.equal(got.isnan().all(1), nan_tok) and torch.equal(got.isnan().any(1), nan_tok)
    # a constant row: zero variance, the output is the LayerNorm bias
    x = torch.zeros(b, C, H, W)
    got = _dwconv(x, torch.zeros_like(w), torch.full((C,), 3.0), lg, lb).cpu()
    assert bool(got.isfinite().all()) and torch.allclose(got, lb.expand_as(got), atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W,C", [(2, 7, 9, 192), (1, 5, 4, 384), (2, 2, 3, 768), (1, 100, 168, 192), (1, 25, 42, 768),
                                     (1, 3, 1, 128)])
def test_layernorm_s2d_vs_fp64(b, H, W, C):
    gen = torch.Generator().manual_seed(H * 7 + W + C)
    x = torch.randn(b, C, H, W, generator=gen) * 3 + 1
    x[0, :, 0, 0] = 2.5  # a constant row
    if H * W > 4:
        x[-1, 3, H - 1, W - 2] = float("nan")
    lg, lb = _ln_affine(C, gen)
    got = pkg.cabi.layernorm_tokens_s2d(_rows(x).to(DEV), (H, W), lg.to(DEV), lb.to(DEV)).cpu().double()
    ho, wo = H // 2, W // 2
    assert tuple(got.shape) == (b, ho * wo, 4 * C)
    if ho == 0 or wo == 0:
        return
    ref = _ln64(x.double(), lg, lb)[:, :, :2 * ho, :2 * wo]
    ref = ref.reshape(b, C, ho, 2, wo, 2).permute(0, 2, 4, 3, 5, 1).reshape(b, ho * wo, 4 * C)
    assert torch.equal(got.isnan(), ref.isnan())
    assert float((got - ref).nan_to_num().abs().max()) <= 2e-6 * float(ref.nan_to_num().abs().max())
    assert torch.allclose(got[0, 0, :C], lb.double(), atol=1e-6)


# ---- GPU: the projection GEMM's CNBlock epilogue -------------------------------------------------------------------------
def _split(w):
    return pkg.cabi.split_f16_pair_dev(w.contiguous().to(DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("act", [0, 2])
@pytest.mark.parametrize("use_s", [False, True])
@pytest.mark.parametrize("zmode", ["none", "z", "alias"])
@pytest.mark.parametrize("mag", ["unit", "tiny", "large"])
def test_gemm_ex_vs_fp64(act, use_s, zmode, mag):
    """C = z + s * (act(A) W^T + b) within 2^-17 of sum |act(A)| |W| + |b| (scaled by s) + rounding of z, for activations of
    unit size, below GELU's minimum (max|A| < 0.17) and of size 1e4"""
    gen = torch.Generator().manual_seed(act * 100 + use_s * 10 + len(zmode) + len(mag))
    M, K, N = 333, 768, 192
    amp = {"unit": 1.0, "tiny": 0.1, "large": 1e4}[mag]
    a = torch.randn(M, K, generator=gen) * amp
    if mag == "tiny":
        a = a.clamp(-0.16, 0.16)
    w = torch.randn(N, K, generator=gen) / K ** 0.5
    bias = torch.randn(N, generator=gen) * 0.1
    s = 0.05 + torch.rand(N, generator=gen) if use_s else None
    z = torch.randn(M, N, generator=gen) * 2
    ad = a.to(DEV)
    kw = dict(act=act, col_scale=s.to(DEV) if s is not None else None)
    if zmode == "z":
        zd = z.to(DEV)
        got = pkg.cabi.gemm_f16x3_ex(ad, pkg.cabi.pow2_scale(ad, 12), *_split(w), bias.to(DEV), z=zd, **kw)
        assert torch.equal(zd.cpu(), z)
    elif zmode == "alias":
        zd = z.to(DEV)
        got = pkg.cabi.gemm_f16x3_ex(ad, pkg.cabi.pow2_scale(ad, 12), *_split(w), bias.to(DEV), z=zd, out=zd, **kw)
        assert got is zd
    else:
        got = pkg.cabi.gemm_f16x3_ex(ad, pkg.cabi.pow2_scale(ad, 12), *_split(w), bias.to(DEV), **kw)
    a64 = F.gelu(a.double()) if act == 2 else a.double()
    y = a64 @ w.double().t() + bias.double()
    bnd = a64.abs() @ w.double().abs().t() + bias.double().abs()
    if s is not None:
        y, bnd = y * s.double(), bnd * s.double()
    if zmode != "none":
        y, bnd = y + z.double(), bnd + z.double().abs()
    err = (got.cpu().double() - y).abs()
    assert bool((err <= 2.0 ** -17 * bnd + 2.0 ** -22 * float(bnd.max())).all()), float(err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,N", [(2 * 5000, 256, 256), (300, 256, 1024), (2 * 1050, 1024, 256), (8, 256, 91), (2 * 300, 256, 256)])
def test_scaled_entry_point_bit_identical_to_ex_with_options_off(M, K, N):
    """sdetr_gemm_f16x3_scaled and sdetr_gemm_f16x3_ex without activation, column scale or residual write the same bits, at
    the projection shapes of the encoder; sdetr_gemm_f16x3_pre with a GELU equals ex with GELU and both scales 2^4 / w_scale"""
    gen = torch.Generator().manual_seed(M + K + N)
    a = torch.randn(M, K, generator=gen).to(DEV)
    w = torch.randn(N, K, generator=gen) / K ** 0.5
    bias = (torch.randn(N, generator=gen) * 0.1).to(DEV)
    w_hi, w_lo, w_scale = _split(w)
    s = pkg.cabi.pow2_scale(a, 12)
    old = pkg.cabi.gemm_f16x3_scaled(a, s, w_hi, w_lo, w_scale, bias)
    new = pkg.cabi.gemm_f16x3_ex(a, s, w_hi, w_lo, w_scale, bias)
    assert torch.equal(old, new)
    hi, lo, host_scale = pkg.cabi.split_f16_pair(w.to(DEV))
    pre = pkg.cabi.gemm_f16x3_pre(a, hi, lo, host_scale, bias, act=2)
    ex = pkg.cabi.gemm_f16x3_ex(a, torch.full((1,), 16.0, device=DEV), hi, lo, torch.full((1,), host_scale, device=DEV), bias,
                                act=2)
    assert torch.equal(pre.reshape(ex.shape), ex)


# ---- GPU: forward_tokens --------------------------------------------------------------------------------------------------
FWD_CASES = {
    "l_64x96": ("conv_l", (1, 2, 3), 1, 64, 96),
    "l_ragged_all": ("conv_l", (0, 1, 2, 3), 3, 200, 312),
    "l_config2": ("conv_l", (1, 2, 3), 2, 800, 1344),
    "b_97x131_all": ("conv_b", (0, 1, 2, 3), 2, 97, 131),
    "b_ragged": ("conv_b", (1, 2, 3), 3, 200, 312),
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
    assert list(tok) == [f"features.{2 * i + 1}" for i in ri]
    for k, (e_tok, e_fp32, e_tf32) in errs.items():
        print(f"{case} {k}: tokens {e_tok:.3e}  torch fp32 {e_fp32:.3e}  TF32 {e_tf32:.3e}")
        assert e_tok <= 16 * e_fp32 and e_tok < 0.1 * e_tf32, (k, e_tok, e_fp32, e_tf32)
    for k, v in tok.items():
        bb, c, h, w = v.shape
        assert v.stride() == (h * w * c, 1, w * c, c) and v.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.gpu
def test_golden_outputs_on_gpu():
    check_golden_outputs_on_gpu(_backbone(), "convnext_l_backbone")


@pytest.mark.gpu
def test_no_sync_graph_replay_repeatability_and_launches():
    m = _backbone().to(DEV)
    x = padded_images(2, 97, 131, torch.Generator().manual_seed(3)).to(DEV)
    check_no_sync_graph_replay_repeatability_and_launches(m, x, 190)


@pytest.mark.gpu
def test_kernel_weights_follow_parameter_changes():
    m = _backbone().to(DEV)
    x = padded_images(1, 64, 96, torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        a = m(x)["features.7"].clone()
        m.features[5][3].layer_scale.mul_(2.0)
        b = m(x)["features.7"].clone()
        m.features[3][1].block[2].weight.mul_(0.5)
        c = m(x)["features.7"]
        want = copy.deepcopy(m).double()(x.double())["features.7"]
    assert not torch.equal(a, b) and not torch.equal(b, c)
    assert rel_err(c, want) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["input_grad", "param_grad", "stochastic_depth", "conv_t", "gelu_tanh"])
def test_torch_path_on_cuda_is_the_op_chain(name):
    arch = "conv_t" if name == "conv_t" else "conv_b"
    m = CNB(arch, return_indices=(1, 2, 3), freeze_indices=(0, 1, 2, 3) if name != "param_grad" else (0,)).to(DEV).eval()
    x = padded_images(1, 64, 96, torch.Generator().manual_seed(5)).to(DEV)
    if name == "gelu_tanh":
        m.features[3][0].block[4] = nn.GELU(approximate="tanh")
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
    """images -> ConvNeXt (channels-last views) -> ChannelMapper(in_channels=num_channels) with zero transposes ->
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
