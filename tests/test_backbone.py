"""ResNetBackbone and FrozenBatchNorm2d (backbone.py): the torch mirror against the UNMODIFIED reference
(tests/golden/resnet50_backbone.npz, made by tools/make_backbone_golden.py) and the constructor on the CPU; the stem, max-pool
and residual / ReLU convolution epilogue kernels, forward_tokens and the backbone -> ChannelMapper -> encoder chain on the GPU."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import salience_detr_b200 as pkg
from backbone_harness import (DEV, FBN, chain_graph_matches_eager, check_no_sync_graph_replay_repeatability_and_launches,
                              check_weight_loading, errors, golden, mapper_chain, rel_err, resnet_backbone, resnet_images,
                              resnet_weights, tf32)


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_state_dict_init_and_freeze_match_reference():
    g = golden("resnet50_backbone")
    m = resnet_backbone()
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["shapes_json"]
    assert len(g["shapes_json"]) == 265 and not any(k.startswith("fc.") for k in g["shapes_json"])
    assert {k: p.requires_grad for k, p in m.named_parameters()} == g["grad_json"]
    assert not m.conv1.training and not m.bn1.training and not m.layer1.training and m.layer2.training
    assert m.num_channels == g["num_channels_json"] == [512, 1024, 2048]
    torch.manual_seed(0)
    init = pkg.ResNetBackbone("resnet50", norm_layer=FBN)
    got = {k: float(v.double().sum()) for k, v in init.state_dict().items()}
    assert got.keys() == g["init_sums_json"].keys()
    assert all(got[k] == v for k, v in g["init_sums_json"].items())


def test_torch_forward_matches_reference():
    g = golden("resnet50_backbone")
    m = resnet_backbone().eval()
    with torch.no_grad():
        outs = m(g["image"])
    assert list(outs) == ["layer2", "layer3", "layer4"]
    for k, v in outs.items():
        want = g[f"out.{k}"]
        assert v.shape == want.shape
        assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max()), k


def test_frozen_batch_norm_formula_and_load():
    bn = FBN(8, eps=1e-3)
    sd = {"weight": torch.rand(8) + 0.5, "bias": torch.randn(8), "running_mean": torch.randn(8), "running_var": torch.rand(8) + 0.5,
          "num_batches_tracked": torch.tensor(7)}
    bn.load_state_dict(sd, strict=True)
    assert sorted(bn.state_dict()) == ["bias", "running_mean", "running_var", "weight"]
    x = torch.randn(2, 8, 3, 5)
    scale = sd["weight"].view(1, -1, 1, 1) * (sd["running_var"].view(1, -1, 1, 1) + 1e-3).rsqrt()
    assert torch.equal(bn(x), x * scale + (sd["bias"].view(1, -1, 1, 1) - sd["running_mean"].view(1, -1, 1, 1) * scale))
    assert not list(bn.parameters())


@pytest.mark.parametrize("arch", sorted(pkg.ResNetBackbone.model_arch))
def test_every_arch_builds(arch):
    m = pkg.ResNetBackbone(arch, norm_layer=FBN, return_indices=(0, 1, 2, 3))
    exp = pkg.ResNetBackbone.model_arch[arch]["block"].expansion
    assert m.num_channels == [64 * exp, 128 * exp, 256 * exp, 512 * exp]
    assert not hasattr(m, "fc") and hasattr(m, "layer4")
    with torch.no_grad():
        outs = m(torch.randn(1, 3, 32, 64))
    assert list(outs) == ["layer1", "layer2", "layer3", "layer4"]
    assert [tuple(v.shape) for v in outs.values()] == [(1, c, 8 // 2 ** i, 16 // 2 ** i) for i, c in enumerate(m.num_channels)]


def test_return_indices_and_extractor_truncation():
    m = pkg.ResNetBackbone("resnet50", norm_layer=FBN, return_indices=(2, 0))
    assert m.num_channels == [1024, 256] and not hasattr(m, "layer4")
    with torch.no_grad():
        assert list(m(torch.randn(1, 3, 32, 32))) == ["layer3", "layer1"]


def test_weights_from_dict_model_and_path(tmp_path):
    check_weight_loading(tmp_path, pkg.ResNetBackbone, "resnet50", resnet_weights, dict(norm_layer=FBN),
                         classifier={"fc.weight": torch.zeros(1000, 2048), "fc.bias": torch.zeros(1000)},
                         drop="layer1.0.conv1.weight", resize="bn1.bias",
                         url="https://download.pytorch.org/models/resnet50-11ad3fa6.pth", bad_arch="resnet51")


def test_tokens_supported_false_cases():
    m = resnet_backbone("resnet50", freeze_indices=(0, 1, 2, 3))
    x = torch.randn(1, 3, 32, 32)
    assert not m.tokens_supported(x)  # CPU input
    assert not pkg.ResNetBackbone("resnext50_32x4d", norm_layer=FBN).layers_supported()
    assert not pkg.ResNetBackbone("resnet50", norm_layer=FBN, replace_stride_with_dilation=[False, False, True]).layers_supported()
    assert not pkg.ResNetBackbone("resnet50").layers_supported()  # nn.BatchNorm2d
    assert not pkg.ResNetBackbone("resnet18", norm_layer=FBN).layers_supported()  # BasicBlock
    assert not pkg.ResNetBackbone("resnet50", norm_layer=FBN, stage_with_dcn=[False, True, False, False]).layers_supported()
    assert m.layers_supported() and resnet_backbone("wide_resnet50_2").layers_supported()


# ---- GPU: kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W", [(1, 97, 131), (2, 64, 96), (3, 33, 47), (1, 5, 7), (2, 1, 1), (1, 7, 200), (2, 300, 3)])
def test_stem_vs_fp64(b, H, W):
    """fp32 FMAs over 147 taps: |err| <= 160 * 2^-24 * (|x| conv |W| + |bias|), the bound of a sequential fp32 sum"""
    gen = torch.Generator().manual_seed(b * 1000 + H * 7 + W)
    x = resnet_images(b, H, W, gen)
    w = torch.randn(64, 3, 7, 7, generator=gen) * (2 / 147) ** 0.5
    bias = torch.randn(64, generator=gen) * 0.5
    got = pkg.cabi.resnet_stem(x.to(DEV), w.reshape(64, 147).t().contiguous().to(DEV), bias.to(DEV))
    ref = F.relu(F.conv2d(x.double(), w.double(), bias.double(), 2, 3))
    bnd = F.conv2d(x.double().abs(), w.double().abs(), bias.double().abs(), 2, 3)
    ho, wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    assert ref.shape[2:] == (ho, wo)
    got = got.cpu().double().view(b, ho, wo, 64).permute(0, 3, 1, 2)
    assert bool(((got - ref).abs() <= 160 * 2.0 ** -24 * bnd + 1e-30).all())


@pytest.mark.gpu
def test_stem_nan_propagates():
    x = torch.zeros(1, 3, 20, 20)
    x[0, 1, 9, 9] = float("nan")
    w = torch.full((147, 64), -1.0)  # every output negative before the ReLU: only the NaN survives it
    got = pkg.cabi.resnet_stem(x.to(DEV), w.to(DEV), torch.full((64,), -1.0, device=DEV)).cpu().view(10, 10, 64)
    ref = F.relu(F.conv2d(x, w.t().reshape(64, 3, 7, 7), torch.full((64,), -1.0), 2, 3))[0].permute(1, 2, 0)
    assert torch.equal(got.isnan(), ref.isnan()) and int(got.isnan().any(-1).sum()) == 16
    assert torch.equal(got.nan_to_num(), ref.nan_to_num())


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W,C", [(1, 97, 131, 64), (3, 20, 33, 64), (2, 1, 1, 64), (1, 2, 7, 256), (2, 5, 3, 8), (1, 200, 336, 64)])
def test_maxpool_vs_torch(b, H, W, C):
    """a maximum is exact: the pool equals torch's max_pool2d bit for bit, NaN where a window holds a NaN"""
    gen = torch.Generator().manual_seed(H * 31 + W + C)
    x = torch.randn(b, C, H, W, generator=gen)
    x[x > 2.5] = float("nan")
    x[-1, C // 2, H // 2, W // 2] = float("nan")
    x[0, :, 0, 0] = float("-inf")
    rows = x.permute(0, 2, 3, 1).reshape(b, H * W, C).contiguous().to(DEV)
    got = pkg.cabi.maxpool3x3s2_tokens(rows, (H, W)).cpu()
    ref = F.max_pool2d(x.double(), 3, 2, 1).float()
    ho, wo = ref.shape[2:]
    got = got.view(b, ho, wo, C).permute(0, 3, 1, 2)
    assert torch.equal(got.isnan(), ref.isnan()) and bool(ref.isnan().any())
    assert torch.equal(got.nan_to_num(), ref.nan_to_num())


def _rows(x):
    b, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(b, h * w, c).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("k,stride,cin,cout", [(1, 1, 64, 256), (3, 2, 128, 128), (1, 2, 256, 512), (3, 1, 64, 64)])
@pytest.mark.parametrize("mode", ["relu", "residual", "alias"])
def test_conv_epilogue_vs_fp64(k, stride, cin, cout, mode):
    """y = act(conv(x, W) + bias + z) with ReLU; with a residual z; with z the output tensor itself.  Bound of the neck's
    convolution test: 2^-17 * (|x| conv |W|) + |z| rounding."""
    gen = torch.Generator().manual_seed(k * 100 + stride * 10 + cin + cout)
    b, h, w = 2, 13, 21
    x = torch.randn(b, cin, h, w, generator=gen)
    wt = torch.randn(cout, cin, k, k, generator=gen) / (cin * k * k) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    z = torch.randn(b, cout, ho, wo, generator=gen)
    w_hi, w_lo, w_scale = pkg.cabi.split_f16_pair_dev(wt.permute(0, 2, 3, 1).contiguous().to(DEV))
    xr = _rows(x).to(DEV)
    ref = F.conv2d(x.double(), wt.double(), bias.double(), stride, k // 2)
    bnd = F.conv2d(x.double().abs(), wt.double().abs(), bias.double().abs(), stride, k // 2)
    args = (xr, (h, w), pkg.cabi.pow2_scale(xr, 12), w_hi, w_lo, w_scale, bias.to(DEV), 1, k, stride, pkg.cabi.ACT_RELU)
    if mode == "relu":
        got = pkg.cabi.conv2d_f16x3(*args)
    elif mode == "residual":
        zr = _rows(z).to(DEV)
        zc = zr.clone()
        got = pkg.cabi.conv2d_f16x3(*args, z=zr)
        assert torch.equal(zr, zc)
        ref, bnd = ref + z.double(), bnd + z.double().abs()
    else:
        got = _rows(z).to(DEV)
        assert pkg.cabi.conv2d_f16x3(*args, out=got, z=got) is got
        ref, bnd = ref + z.double(), bnd + z.double().abs()
    ref = F.relu(ref)
    got = got.cpu().double().view(b, ho, wo, cout).permute(0, 3, 1, 2)
    assert bool(((got - ref).abs() <= 2.0 ** -17 * bnd + 1e-30).all()), float((got - ref).abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("k,stride,groups,c,act", [(3, 1, 4, 256, 3), (3, 2, 1, 256, 3), (1, 1, 1, 512, 3), (1, 1, 1, 256, 0),
                                                   (3, 1, 4, 256, 0)])
def test_conv_zero_residual_bit_identical(k, stride, groups, c, act):
    """sdetr_conv2d_f16x3 with z = NULL (the neck's and the mapper's calls) and with z = 0 write the same bits, at the neck's
    shapes (config-2 level 1: 50 x 84, C 256, groups 4)"""
    gen = torch.Generator().manual_seed(k + 10 * stride + groups + c + act)
    b, h, w = 2, 50, 84
    x = torch.randn(b, h * w, c, generator=gen).to(DEV)
    wt = torch.randn(c, c // groups, k, k, generator=gen) / (c // groups * k * k) ** 0.5
    bias = (torch.randn(c, generator=gen) * 0.1).to(DEV)
    w_hi, w_lo, w_scale = pkg.cabi.split_f16_pair_dev(wt.permute(0, 2, 3, 1).contiguous().to(DEV))
    s = pkg.cabi.pow2_scale(x, 12)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    old = torch.full((b, ho * wo, c), float("nan"), device=DEV)
    rc = pkg.cabi.lib().sdetr_conv2d_f16x3(x.data_ptr(), x.stride(0), x.stride(1), b, h, w, c, s.data_ptr(), w_hi.data_ptr(),
                                           w_lo.data_ptr(), w_scale.data_ptr(), bias.data_ptr(), None, 0, 0, c, groups, k, stride,
                                           act, old.data_ptr(), old.stride(0), old.stride(1), pkg.cabi._stream())
    assert rc == 0
    new = pkg.cabi.conv2d_f16x3(x, (h, w), s, w_hi, w_lo, w_scale, bias, groups, k, stride, act)
    zero = pkg.cabi.conv2d_f16x3(x, (h, w), s, w_hi, w_lo, w_scale, bias, groups, k, stride, act, z=torch.zeros_like(old))
    assert torch.equal(old, new) and torch.equal(old, zero)


# ---- GPU: forward_tokens ------------------------------------------------------------------------------------------------
FWD_CASES = {
    "r50_64x96": ("resnet50", 1, 64, 96),
    "r50_97x131": ("resnet50", 2, 97, 131),
    "r50_ragged": ("resnet50", 3, 120, 168),
    "r50_config2": ("resnet50", 2, 800, 1344),
    "wide50_97x131": ("wide_resnet50_2", 1, 97, 131),
    "r101_64x96": ("resnet101", 2, 64, 96),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(FWD_CASES))
def test_forward_tokens_vs_fp64(case):
    """Every output within 16x the error of the same forward() on cuDNN fp32 (TF32 off), measured here, and below TF32's."""
    arch, b, H, W = FWD_CASES[case]
    m = resnet_backbone(arch, return_indices=(0, 1, 2, 3)).to(DEV)
    x = resnet_images(b, H, W, torch.Generator().manual_seed(H + W)).to(DEV)
    with torch.no_grad():
        assert m.tokens_supported(x)
    errs, tok = errors(m, x)
    for k, (e_tok, e_fp32, e_tf32) in errs.items():
        print(f"{case} {k}: tokens {e_tok:.3e}  cuDNN fp32 {e_fp32:.3e}  TF32 {e_tf32:.3e}")
        assert e_tok <= 16 * e_fp32 and e_tok < e_tf32, (k, e_tok, e_fp32, e_tf32)
    for k, v in tok.items():
        bb, c, h, w = v.shape
        assert v.stride() == (h * w * c, 1, w * c, c) and v.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.gpu
def test_no_sync_graph_replay_repeatability_and_launches():
    m = resnet_backbone(return_indices=(0, 1, 2, 3)).to(DEV)
    x = resnet_images(2, 97, 131, torch.Generator().manual_seed(3)).to(DEV)
    check_no_sync_graph_replay_repeatability_and_launches(m, x, 2 + 2 * 52 - 4)


@pytest.mark.gpu
def test_folded_weights_follow_buffer_changes():
    m = resnet_backbone().to(DEV)
    x = resnet_images(1, 64, 96, torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        a = m(x)["layer4"].clone()
        m.layer3[1].bn2.running_var.mul_(2.0)
        b = m(x)["layer4"]
        want = copy.deepcopy(m).double()(x.double())["layer4"]
    assert not torch.equal(a, b)
    assert rel_err(b, want) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["input_grad", "param_grad", "batchnorm", "resnext", "basic", "dilation"])
def test_torch_path_on_cuda_is_the_op_chain(name):
    kw = dict(arch="resnet50", freeze_indices=(0, 1, 2, 3))
    if name == "param_grad":
        kw["freeze_indices"] = (0,)
    elif name == "batchnorm":
        kw["norm_layer"] = nn.BatchNorm2d
    elif name == "resnext":
        kw["arch"] = "resnext50_32x4d"
    elif name == "basic":
        kw["arch"] = "resnet18"
    elif name == "dilation":
        kw["replace_stride_with_dilation"] = [False, False, True]
    arch = kw.pop("arch")
    m = pkg.ResNetBackbone(arch, return_indices=(1, 2, 3), norm_layer=kw.pop("norm_layer", FBN), **kw).to(DEV).eval()
    x = resnet_images(1, 64, 96, torch.Generator().manual_seed(5)).to(DEV)
    if name == "input_grad":
        x.requires_grad_(True)
    ctx = torch.enable_grad() if name in ("input_grad", "param_grad") else torch.no_grad()
    with ctx:
        assert not m.tokens_supported(x)
        n0 = pkg.cabi.launch_count()
        got = m(x)
        assert pkg.cabi.launch_count() == n0
        want = m.forward_torch(x)
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in got)


# ---- GPU: backbone -> ChannelMapper -> encoder ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_backbone_mapper_encoder_chain():
    """images -> backbone (channels-last views) -> ChannelMapper with zero transposes -> forward_encoder: the memory within 16x
    the error of the cuDNN fp32 backbone chain against the float64 backbone chain, and the whole chain in one CUDA graph"""
    bb = resnet_backbone().to(DEV)
    c = mapper_chain(bb)
    with torch.no_grad():
        ref = c.tr.forward_encoder(c.mapper({k: v.float() for k, v in c.ref_feats.items()}), c.masks, c.pos, plan=c.plan)[0]
        with tf32(False):
            fp32_feats = bb.forward_torch(c.x)
            fp32 = c.tr.forward_encoder(c.mapper(fp32_feats), c.masks, c.pos, plan=c.plan)[0]
        fp32_mapped = c.mapper.forward_tokens(fp32_feats)[0]
    # the mapper's tokens: a smooth function of the backbone's maps
    e_tok, e_fp32 = rel_err(c.mapped, c.ref_mapped.double()), rel_err(fp32_mapped, c.ref_mapped.double())
    print(f"mapper tokens: backbone tokens {e_tok:.3e}, cuDNN fp32 {e_fp32:.3e}")
    assert e_tok <= 16 * e_fp32
    # the memory: its salience top-k can pick other tokens under any rounding difference, so both chains are measured
    e_tok, e_fp32 = rel_err(c.mem, ref.double()), rel_err(fp32, ref.double())
    print(f"encoder memory: backbone tokens {e_tok:.3e}, cuDNN fp32 {e_fp32:.3e}")
    assert e_tok <= 16 * e_fp32
    assert chain_graph_matches_eager(bb, c)
