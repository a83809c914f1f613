"""SwinTransformerBackbone (swin.py): the reference's structure, initialisation, freezing and outputs on the CPU (fixture
tests/golden/swin_l_backbone.npz, made by tools/make_swin_golden.py from the reference itself), a float64 restatement of the
window-attention kernel's index arithmetic against the reference's shifted_window_attention, and on the H100 the token path's
kernels and the module against float64."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F
from torch import nn
from torchvision.models.swin_transformer import _patch_merging_pad

import salience_detr_b200 as pkg
from salience_detr_b200 import swin as swm
from backbone_harness import (DEV, chain_graph_matches_eager, check_golden_outputs_on_gpu,
                              check_no_sync_graph_replay_repeatability_and_launches, check_weight_loading, errors, golden,
                              mapper_chain, padded_images, rel_err, swin_weights, tf32)
from backbone_harness import swin_backbone as _backbone

STB = pkg.SwinTransformerBackbone
TOKEN_ARCHS = ("swin_b", "swin_l", "swin_b_384", "swin_l_384")


# ---- CPU: the module against the reference --------------------------------------------------------------------------------
def test_state_dict_init_and_freeze_match_reference():
    g = golden("swin_l_backbone")
    m = _backbone()
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == g["shapes_json"]
    assert len(g["shapes_json"]) == 349 and sum(k.endswith("relative_position_index") for k in g["shapes_json"]) == 24
    assert not any(k.startswith(("norm.", "head.")) for k in g["shapes_json"])
    assert {k: p.requires_grad for k, p in m.named_parameters()} == g["grad_json"]
    assert m.num_channels == g["num_channels_json"] == [384, 768, 1536]
    m = STB("swin_l", return_indices=(1, 2, 3), freeze_indices=(0,))
    assert not m.features[0].training and not m.features[1].training and not m.features[2].training and m.features[3].training
    torch.manual_seed(0)
    init = STB("swin_l")
    got = {k: float(v.double().sum()) for k, v in init.state_dict().items()}
    assert got.keys() == g["init_sums_json"].keys()
    assert all(got[k] == v for k, v in g["init_sums_json"].items())


def test_torch_forward_matches_reference():
    g = golden("swin_l_backbone")
    m = _backbone()
    with torch.no_grad():
        outs = m(g["image"])
    assert list(outs) == ["features.3", "features.5", "features.7"]
    for k, v in outs.items():
        want = g[f"out.{k}"]
        assert v.shape == want.shape
        assert v.is_contiguous(memory_format=torch.channels_last)  # the reference's permute of a BHWC tensor, as it is
        assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max()), k


@pytest.mark.parametrize("arch", sorted(STB.model_arch))
def test_every_arch_builds(arch):
    m = STB(arch)
    cfg = STB.model_arch[arch]
    assert m.num_channels == [cfg["embed_dim"] * 2 ** i for i in range(4)]
    assert not hasattr(m, "norm") and not hasattr(m, "head") and len(m.features) == 8
    assert [len(m.features[2 * i + 1]) for i in range(4)] == list(cfg["depths"])
    blocks = [blk for i in range(4) for blk in m.features[2 * i + 1]]
    assert blocks[0].stochastic_depth.p == 0 and blocks[-1].stochastic_depth.p == pytest.approx(cfg["stochastic_depth_prob"])
    assert [list(b.attn.shift_size) for b in blocks[:2]] == [[0, 0], [w // 2 for w in cfg["window_size"]]]
    with torch.no_grad():
        outs = m(torch.randn(1, 3, 64, 96))
    assert [tuple(v.shape) for v in outs.values()] == [(1, c, math.ceil(16 / 2 ** i), math.ceil(24 / 2 ** i))
                                                       for i, c in enumerate(m.num_channels)]
    assert m.layers_supported() == (arch in TOKEN_ARCHS)


def test_return_indices_and_extractor_truncation():
    m = STB("swin_b", return_indices=(2, 0))
    assert m.num_channels == [512, 128] and len(m.features) == 6
    assert not any(k.startswith(("features.6", "features.7")) for k in m.state_dict())
    with torch.no_grad():
        assert list(m(torch.randn(1, 3, 32, 32))) == ["features.5", "features.1"]
    m = STB("swin_b", return_indices=(0,))
    assert len(m.features) == 2 and m.launches_per_forward() == 1 + 11 * 2
    assert _backbone("swin_l").launches_per_forward() == 274


def test_kwargs_work_as_in_reference():
    m = STB("swin_b", stochastic_depth_prob=0.1, mlp_ratio=2.0, return_indices=(0, 1, 2, 3))
    assert m.features[7][-1].stochastic_depth.p == pytest.approx(0.1) and m.features[1][0].mlp[0].out_features == 256
    m = STB("swin_b", window_size=None, return_indices=(0,))  # None keeps the arch's value, as in the reference
    assert list(m.features[1][1].attn.window_size) == [7, 7]
    m = STB("swin_b", window_size=[8, 6], return_indices=(0,))
    assert list(m.features[1][1].attn.shift_size) == [4, 3] and m.layers_supported()
    m = STB("swin_b", dropout=0.1, attention_dropout=0.1, return_indices=(0,))
    assert m.features[1][0].attn.dropout == 0.1 and m.features[1][0].attn.attention_dropout == 0.1
    m = STB("swin_b", block=swm.SwinTransformerBlockV2, downsample_layer=swm.PatchMergingV2, return_indices=(0, 1))
    assert type(m.features[1][0]) is swm.SwinTransformerBlockV2 and not m.layers_supported()
    with pytest.raises(TypeError, match="unexpected keyword"):
        STB("swin_b", layer_scale=0.5)


def test_weights_from_dict_model_and_path(tmp_path):
    check_weight_loading(tmp_path, STB, "swin_b", swin_weights, {},
                         classifier={"norm.weight": torch.ones(1024), "norm.bias": torch.zeros(1024),
                                     "head.weight": torch.zeros(1000, 1024), "head.bias": torch.zeros(1000)},
                         drop="features.1.0.attn.relative_position_index", resize="features.0.0.bias",
                         url="https://download.pytorch.org/models/swin_b-68c6b09e.pth", bad_arch="swin_xl")


def test_tokens_supported_false_cases():
    m = STB("swin_b", freeze_indices=(0, 1, 2, 3))
    assert m.layers_supported()
    assert not m.tokens_supported(torch.randn(1, 3, 64, 64))  # CPU input
    assert not STB("swin_t").layers_supported() and not STB("swin_s").layers_supported()  # 96-wide stages
    assert not STB("swin_v2_t").layers_supported() and not STB("swin_v2_b").layers_supported()
    m = STB("swin_b", return_indices=(0,))
    m.features[1][0].mlp[1] = nn.GELU(approximate="tanh")
    assert not m.layers_supported()
    m = STB("swin_b", return_indices=(0,), window_size=[13, 12])  # 156 tokens per window
    assert not m.layers_supported()


# ---- CPU: the kernel's index arithmetic, restated in float64 ---------------------------------------------------------------
def window_attention_restated(qkv, hw, qkv_bias, rel_bias, heads, window, shift):
    """What sdetr_window_attention_tokens computes, in torch: qkv (b, H*W, 3C) rows gathered by source index (pad positions read
    the qkv bias), the shift disabled where the window covers the padded map, region ids from the rolled frame, -100 added
    between regions, and each query's output written back to its source pixel -> (b, H*W, C)"""
    b, n, c3 = qkv.shape
    C, (H, W), (wh, ww) = c3 // 3, hw, window
    pad_H, pad_W = -(-H // wh) * wh, -(-W // ww) * ww
    sh = 0 if wh >= pad_H else shift[0]
    sw = 0 if ww >= pad_W else shift[1]
    nwy, nwx, N = pad_H // wh, pad_W // ww, wh * ww
    R = (torch.arange(nwy)[:, None, None, None] * wh + torch.arange(wh)[None, None, :, None]).expand(nwy, nwx, wh, ww)
    Cc = (torch.arange(nwx)[None, :, None, None] * ww + torch.arange(ww)[None, None, None, :]).expand(nwy, nwx, wh, ww)
    R, Cc = R.reshape(nwy * nwx, N), Cc.reshape(nwy * nwx, N)
    sr, sc = (R + sh) % pad_H, (Cc + sw) % pad_W
    valid = (sr < H) & (sc < W)
    src = torch.where(valid, sr * W + sc, n)
    rows = torch.cat([qkv, qkv_bias.expand(b, 1, c3)], 1)
    g = rows[:, src.flatten()].view(b, nwy * nwx, N, 3, heads, C // heads).permute(3, 0, 1, 4, 2, 5)
    q, k, v = g[0], g[1], g[2]
    logits = (q * (C // heads) ** -0.5) @ k.transpose(-1, -2) + rel_bias

    def region(p, pad, w, s):
        return torch.where(p < pad - w, 0, torch.where(p < pad - s, 1, 2))

    reg = 3 * region(R, pad_H, wh, sh) + region(Cc, pad_W, ww, sw)
    logits = logits + torch.where(reg[:, :, None] == reg[:, None, :], 0.0, -100.0).to(logits.dtype)[None, :, None]
    out = (logits.softmax(-1) @ v).permute(0, 1, 3, 2, 4).reshape(b, nwy * nwx * N, C)
    y = torch.zeros(b, n, C, dtype=qkv.dtype)
    y[:, src.flatten()[valid.flatten()]] = out[:, valid.flatten()]
    return y


# (b, H, W, heads, window): multiples of the window, not multiples, smaller than it in one or both dimensions
ATT_CASES = [
    (1, 14, 21, 1, (7, 7)), (2, 16, 25, 6, (7, 7)), (3, 8, 13, 12, (7, 7)), (1, 4, 7, 24, (7, 7)), (2, 2, 4, 48, (7, 7)),
    (2, 9, 5, 4, (7, 7)), (1, 24, 36, 2, (12, 12)), (2, 25, 30, 8, (12, 12)), (1, 13, 7, 3, (12, 12)), (3, 5, 9, 16, (12, 12)),
    (1, 1, 1, 1, (7, 7)), (2, 20, 3, 5, (7, 7)),
]


def _att_inputs(b, H, W, heads, window, gen, dtype=torch.float64, amp=1.0):
    C, N = 32 * heads, window[0] * window[1]
    x = torch.randn(b, H, W, C, generator=gen, dtype=dtype)
    wqkv = torch.randn(3 * C, C, generator=gen, dtype=dtype) / C ** 0.5 * amp
    bqkv = torch.randn(3 * C, generator=gen, dtype=dtype) * amp
    rel = torch.randn(heads, N, N, generator=gen, dtype=dtype) * 2
    return x, wqkv, bqkv, rel


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("case", range(len(ATT_CASES)))
def test_restated_index_arithmetic_is_the_reference(case, shifted):
    b, H, W, heads, window = ATT_CASES[case]
    gen = torch.Generator().manual_seed(case * 2 + shifted)
    x, wqkv, bqkv, rel = _att_inputs(b, H, W, heads, window, gen, amp=2.0)
    C = 32 * heads
    shift = [w // 2 for w in window] if shifted else [0, 0]
    want = swm.shifted_window_attention(x, wqkv, torch.eye(C, dtype=torch.float64), rel[None], list(window), heads, shift,
                                        qkv_bias=bqkv, training=False)
    qkv = x.reshape(b, H * W, C) @ wqkv.t() + bqkv
    got = window_attention_restated(qkv, (H, W), bqkv, rel, heads, window, shift)
    assert torch.allclose(got, want.reshape(b, H * W, C), rtol=1e-10, atol=1e-10)


def test_restated_nan_pattern_is_the_reference():
    """a NaN pixel poisons every query of its window, other regions behind the -100 mask included, and nothing else"""
    b, H, W, heads, window = 1, 16, 25, 2, (7, 7)
    x, wqkv, bqkv, rel = _att_inputs(b, H, W, heads, window, torch.Generator().manual_seed(3))
    x[0, 15, 24] = float("nan")  # in the last rolled window, which holds all four regions
    C, shift = 32 * heads, [3, 3]
    want = swm.shifted_window_attention(x, wqkv, torch.eye(C, dtype=torch.float64), rel[None], list(window), heads, shift,
                                        qkv_bias=bqkv, training=False).reshape(b, H * W, C)
    got = window_attention_restated(x.reshape(b, H * W, C) @ wqkv.t() + bqkv, (H, W), bqkv, rel, heads, window, shift)
    assert torch.equal(got.isnan(), want.isnan())
    assert 4 < int(want.isnan().all(-1).sum()) < H * W and torch.equal(want.isnan().all(-1), want.isnan().any(-1))


# ---- GPU: kernels ---------------------------------------------------------------------------------------------------------
def _kernel_attention(qkv, hw, bqkv, rel, heads, window, shift):
    return pkg.cabi.window_attention_tokens(qkv.float().to(DEV), hw, bqkv.float().to(DEV), rel.float().to(DEV), heads, window,
                                            shift).cpu().double()


@pytest.mark.gpu
@pytest.mark.parametrize("amp", [1.0, 6.0])
@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("case", range(len(ATT_CASES)))
def test_window_attention_vs_fp64(case, shifted, amp):
    """the kernel against the float64 restatement on the same fp32 inputs; amp 6 scales the logits up to where the -100 mask
    and the pad keys change the softmax"""
    b, H, W, heads, window = ATT_CASES[case]
    gen = torch.Generator().manual_seed(100 + case * 2 + shifted)
    x, wqkv, bqkv, rel = _att_inputs(b, H, W, heads, window, gen, dtype=torch.float32, amp=amp)
    C = 32 * heads
    qkv = x.reshape(b, H * W, C) @ wqkv.t() + bqkv
    shift = [w // 2 for w in window] if shifted else [0, 0]
    got = _kernel_attention(qkv, (H, W), bqkv, rel, heads, window, shift)
    want = window_attention_restated(qkv.double(), (H, W), bqkv.double(), rel.double(), heads, window, shift)
    q = qkv[..., :C].double().abs().max()
    lmax = float(q * qkv[..., C:2 * C].double().abs().max() * 32 ** 0.5 + rel.abs().max() + 100)
    vmax = float(max(qkv[..., 2 * C:].abs().max(), bqkv.abs().max()))
    err = float((got - want).abs().max())
    assert err <= 4e-7 * lmax * vmax, (err, lmax, vmax)


@pytest.mark.gpu
@pytest.mark.parametrize("part", ["key", "value"])
def test_window_attention_nan_poisons_what_torch_poisons(part):
    b, H, W, heads, window = 2, 16, 25, 3, (7, 7)
    x, wqkv, bqkv, rel = _att_inputs(b, H, W, heads, window, torch.Generator().manual_seed(7), dtype=torch.float32)
    C = 32 * heads
    qkv = x.reshape(b, H * W, C) @ wqkv.t() + bqkv
    col = (C if part == "key" else 2 * C) + 32 * 1 + 5  # head 1
    qkv[1, 15 * W + 24, col] = float("nan")  # the last rolled window, which holds all four regions
    shift = [3, 3]
    got = _kernel_attention(qkv, (H, W), bqkv, rel, heads, window, shift)
    want = window_attention_restated(qkv.double(), (H, W), bqkv.double(), rel.double(), heads, window, shift)
    assert torch.equal(got.isnan(), want.isnan())
    poisoned = want.isnan().any(-1)
    assert 4 < int(poisoned.sum()) < H * W and not bool(poisoned[0].any())
    ok = ~want.isnan()
    assert float((got[ok] - want[ok]).abs().max()) < 1e-4


def _ln_affine(c, gen):
    return 1 + (torch.rand(c, generator=gen) - 0.5) * 0.5, torch.randn(c, generator=gen) * 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("b,H,W,C", [(2, 16, 25, 192), (1, 7, 9, 384), (2, 8, 13, 768), (1, 1, 1, 768), (3, 3, 1, 256),
                                     (1, 200, 336, 192), (2, 5, 6, 64)])
def test_patch_merge_layernorm_vs_fp64(b, H, W, C):
    gen = torch.Generator().manual_seed(H * 7 + W + C)
    x = torch.randn(b, H, W, C, generator=gen) * 3 + 1
    x[0, :2, :2] = 2.5  # output row (0, 0) constant where the map has 2 x 2 pixels
    if H * W > 4:
        x[-1, H - 1, W - 2, 3] = float("nan")
    lg, lb = _ln_affine(4 * C, gen)
    got = pkg.cabi.patch_merge_layernorm_tokens(x.reshape(b, H * W, C).to(DEV), (H, W), lg.to(DEV), lb.to(DEV)).cpu().double()
    ho, wo = (H + 1) // 2, (W + 1) // 2
    assert tuple(got.shape) == (b, ho * wo, 4 * C)
    cat = _patch_merging_pad(x.double())  # the reference's pad and 2x2 concatenation
    ref = F.layer_norm(cat, (4 * C,), lg.double(), lb.double(), 1e-5).reshape(b, ho * wo, 4 * C)
    assert torch.equal(got.isnan(), ref.isnan())
    assert float((got - ref).nan_to_num().abs().max()) <= 2e-6 * float(ref.nan_to_num().abs().max())
    if H >= 2 and W >= 2:
        assert torch.allclose(got[0, 0], lb.double(), atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(1, 64), (333, 192), (1000, 384), (77, 768), (129, 1536), (134400, 192), (5, 1024)])
def test_layernorm_tokens_vs_fp64(rows, C):
    gen = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, C, generator=gen) * 2 + 0.5
    x[0] = 1.25
    if rows > 2:
        x[1, 7] = float("nan")
        x[2] = 1e4 + torch.randn(C, generator=gen) * 1e-2
    lg, lb = _ln_affine(C, gen)
    got = pkg.cabi.layernorm_tokens(x.to(DEV), lg.to(DEV), lb.to(DEV), 1e-5).cpu().double()
    ref = F.layer_norm(x.double(), (C,), lg.double(), lb.double(), 1e-5)
    assert torch.equal(got.isnan(), ref.isnan())
    assert torch.allclose(got[0], lb.double(), atol=1e-6)
    # fp32 rounds the mean to |mean| * 2^-24: relative to the row's spread that grows with |mean| / std
    xd = x.double()
    bound = 1e-5 * (1 + xd.mean(1).abs() / (xd.std(1, correction=0) + 1e-3))
    err = (got - ref).nan_to_num().abs().amax(1)
    assert bool((err <= bound.nan_to_num()).all()), float((err / bound).nan_to_num().max())


# ---- GPU: forward_tokens --------------------------------------------------------------------------------------------------
FWD_CASES = {
    "l_64x100": ("swin_l", (1, 2, 3), 2, 64, 100),
    "l_ragged_all": ("swin_l", (0, 1, 2, 3), 3, 200, 312),
    "l_config2": ("swin_l", (1, 2, 3), 2, 800, 1344),
    "b_97x131_all": ("swin_b", (0, 1, 2, 3), 2, 97, 131),
    "l384_ragged": ("swin_l_384", (1, 2, 3), 2, 150, 230),
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
        assert v._base is not None and v._base.shape == (bb, h * w, c)  # a view of its own token buffer
    ptrs = [v.data_ptr() for v in tok.values()]
    assert len(set(ptrs)) == len(ptrs)


@pytest.mark.gpu
def test_golden_outputs_on_gpu():
    check_golden_outputs_on_gpu(_backbone(), "swin_l_backbone")


@pytest.mark.gpu
def test_no_sync_graph_replay_repeatability_and_launches():
    m = _backbone().to(DEV)
    x = padded_images(2, 97, 131, torch.Generator().manual_seed(3)).to(DEV)
    check_no_sync_graph_replay_repeatability_and_launches(m, x, 274)


@pytest.mark.gpu
def test_kernel_weights_follow_parameter_changes():
    m = _backbone().to(DEV)
    x = padded_images(1, 64, 100, torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        outs = [m(x)["features.7"].clone()]
        m.features[5][3].attn.relative_position_bias_table.mul_(-1.0)
        outs.append(m(x)["features.7"].clone())
        m.features[3][1].norm2.weight.mul_(0.5)
        outs.append(m(x)["features.7"].clone())
        m.features[7][0].attn.qkv.weight.mul_(1.5)
        outs.append(m(x)["features.7"])
        want = copy.deepcopy(m).double()(x.double())["features.7"]
    assert all(not torch.equal(a, b) for a, b in zip(outs, outs[1:]))
    assert rel_err(outs[-1], want) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["input_grad", "param_grad", "stochastic_depth", "swin_t", "swin_v2_t"])
def test_torch_path_on_cuda_is_the_op_chain(name):
    arch = name if name.startswith("swin_") else "swin_b"
    m = STB(arch, return_indices=(1, 2, 3), freeze_indices=(0, 1, 2, 3) if name != "param_grad" else (0,)).to(DEV).eval()
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
    """images -> Swin-L (channels-last views) -> ChannelMapper(in_channels=num_channels) with zero transposes ->
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
