"""ChannelMapper (channel_mapper.py): the torch mirror against the UNMODIFIED reference (tests/golden/channel_mapper.npz, made by
tools/make_channel_mapper_golden.py) on the CPU, the token-layout kernels (sdetr_group_norm_tokens, sdetr_token_lpos_keep),
forward_tokens and the transformer's token-backed features on the GPU."""
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import salience_detr_b200 as pkg
from conftest import GOLDEN
from oracle import make_golden as mg
from oracle import oracle as orc
from tools import make_channel_mapper_golden as mcg
from tools import make_neck_golden as mng

DEV = "cuda:0"


def _golden():
    z = np.load(os.path.join(GOLDEN, "channel_mapper.npz"), allow_pickle=False)
    return {k: (str(z[k]) if z[k].dtype.kind in "US" else torch.from_numpy(z[k])) for k in z.files}


def _torch_chain(mapper, inputs):
    """the reference's forward written with functional ops (conv -> norm -> activation per Conv2dNormActivation)"""
    def block(m, x):
        conv = m[0]
        y = F.conv2d(x, conv.weight, conv.bias, conv.stride, conv.padding, conv.dilation, conv.groups)
        for layer in list(m)[1:]:
            y = layer(y)
        return y

    xs = list(inputs.values())
    outs = [block(mapper.convs[i], xs[i]) for i in range(len(xs))]
    for i in range(len(xs), len(mapper.convs)):
        outs.append(block(mapper.convs[i], xs[-1] if i == len(xs) else outs[-1]))
    return outs


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_state_dict_matches_reference_keys_and_loads_strict():
    g = _golden()
    want = json.loads(g["shapes_json"])
    m = mcg.build(pkg.ChannelMapper)
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == want
    assert "convs.3.0.weight" in want and "convs.0.0.bias" not in want  # GroupNorm: the convs have no bias
    sd = {k: torch.randn(v, generator=torch.Generator().manual_seed(i)) for i, (k, v) in enumerate(sorted(want.items()))}
    fresh = pkg.ChannelMapper(list(mcg.IN_CHANNELS), mcg.OUT_CHANNELS, mcg.NUM_OUTS)
    fresh.load_state_dict(sd, strict=True)
    assert torch.equal(fresh.convs[3][1].bias, sd["convs.3.1.bias"])
    assert fresh.num_channels == [mcg.OUT_CHANNELS] * mcg.NUM_OUTS


def test_detector_checkpoint_loads_with_neck_prefix():
    m = mcg.build(pkg.ChannelMapper)
    src = {k: v + 1.0 for k, v in m.state_dict().items()}
    ckpt = {"model": {**{"neck." + k: v for k, v in src.items()}, "backbone.conv1.weight": torch.zeros(64, 3, 7, 7),
                      "transformer.level_embeds": torch.zeros(4, 256)}}
    res = pkg.load_reference_checkpoint(m, ckpt, prefix="neck.")
    assert res == {"missing": [], "unexpected": [], "mismatched": []}
    assert all(torch.equal(m.state_dict()[k], v) for k, v in src.items())


def test_torch_forward_matches_reference():
    """seeded construction (the reference's xavier initialisation, in the reference's RNG order) + the perturbed affine: the
    four outputs of the reference module"""
    g = _golden()
    m = mcg.build(pkg.ChannelMapper)
    with torch.no_grad():
        outs = m(mcg.inputs())
    assert len(outs) == 4
    for i, o in enumerate(outs):
        assert o.shape == g[f"out{i}"].shape
        assert (o - g[f"out{i}"]).abs().max() < 1e-5, i


EXCLUDED = {
    "activation": dict(activation_layer=nn.ReLU),
    "kernel_size_3": dict(kernel_size=3),
    "width_not_64": dict(in_channels=(96, 256, 512)),
    "batchnorm": dict(norm_layer=nn.BatchNorm2d),
}


def _excluded(name):
    kw = dict(EXCLUDED[name])
    cin = kw.pop("in_channels", mcg.IN_CHANNELS)
    torch.manual_seed(0)
    m = pkg.ChannelMapper(list(cin), mcg.OUT_CHANNELS, mcg.NUM_OUTS, **kw).eval()
    g = torch.Generator().manual_seed(1)
    inputs = OrderedDict((str(i), torch.randn(2, c, h, w, generator=g)) for i, (c, (h, w)) in enumerate(zip(cin, mcg.SHAPES)))
    return m, inputs


@pytest.mark.parametrize("name", sorted(EXCLUDED))
def test_excluded_configurations_fall_back_cpu(name):
    m, inputs = _excluded(name)
    assert not m.layers_supported()
    with torch.no_grad():
        assert not m.tokens_supported(inputs)
        for a, b in zip(m(inputs), _torch_chain(m, inputs)):
            assert torch.allclose(a, b, atol=1e-5, rtol=1e-5)


def test_cpu_inputs_and_training_fall_back():
    m = mcg.build(pkg.ChannelMapper)
    assert m.layers_supported()
    inputs = mcg.inputs()
    assert not m.tokens_supported(inputs)  # CPU
    m.train()
    outs = m(inputs)
    assert all(o.requires_grad for o in outs)
    sum(o.sum() for o in outs).backward()
    assert m.convs[3][0].weight.grad is not None


# ---- GPU: kernels -----------------------------------------------------------------------------------------------------
def _gn_ref64(tok, sizes, gamma, beta, groups, eps):
    b, _, c = tok.shape
    out, s = [], 0
    for l, n in enumerate(sizes):
        x = tok[:, s:s + n].double().cpu().transpose(1, 2)  # (b, C, n)
        out.append(F.group_norm(x, groups, gamma[l].double().cpu(), beta[l].double().cpu(), eps).transpose(1, 2))
        s += n
    return torch.cat(out, 1)


GN_MAPS = [(1, 1), (3, 5), (1, 7), (12, 20), (100, 168)]


@pytest.mark.gpu
@pytest.mark.parametrize("c,groups", [(256, 32), (256, 16), (512, 32), (512, 16), (192, 32)])
@pytest.mark.parametrize("b", [1, 2])
def test_group_norm_kernel_vs_fp64(c, groups, b):
    """levels from 1x1 to 100x168 in a token-range view of a larger buffer (the leading level must stay untouched); the 12x20
    level sits at 1e4 + N(0, 1), where a sum / sum-of-squares variance would lose every significant bit.  Bound: 1e-4 on the
    O(1) outputs, plus, at the offset level, the rounding of an fp32 mean of magnitude 1e4 (4 ulp, times rstd * |gamma|).
    Bit-identical from run to run."""
    gen = torch.Generator().manual_seed(c + groups + b)
    sizes = [h * w for h, w in GN_MAPS]
    lead = 7
    buf = torch.randn(b, lead + sum(sizes), c, generator=gen)
    s_off = lead + sum(sizes[:3])
    buf[:, s_off:s_off + sizes[3]] += 1e4
    buf[:, lead + sum(sizes[:4]):] *= 3.0
    gamma = 1.0 + 0.3 * torch.randn(len(sizes), c, generator=gen)
    beta = 0.3 * torch.randn(len(sizes), c, generator=gen)
    eps = 1e-5
    want = _gn_ref64(buf[:, lead:], sizes, gamma, beta, groups, eps)
    dbuf = buf.to(DEV)
    g, bt = gamma.to(DEV), beta.to(DEV)
    got = pkg.cabi.group_norm_tokens_(dbuf[:, lead:], sizes, g, bt, groups, eps)
    assert got.data_ptr() == dbuf.data_ptr() + lead * c * 4
    assert torch.equal(dbuf[:, :lead].cpu(), buf[:, :lead])
    err = (got.cpu().double() - want).abs()
    tol = torch.full_like(err, 1e-4)
    o0 = sum(sizes[:3])
    tol[:, o0:o0 + sizes[3]] += 4 * 2.0 ** -23 * 1e4 * 1.1 * gamma[3].abs().double()
    assert bool((err <= tol).all()), float(err.max())
    print(f"group_norm_tokens C={c} G={groups} b={b}: max err {float(err.max()):.2e} "
          f"(O(1) levels {float(torch.cat([err[:, :o0], err[:, o0 + sizes[3]:]], 1).max()):.2e})")
    again = buf.to(DEV)
    pkg.cabi.group_norm_tokens_(again[:, lead:], sizes, g, bt, groups, eps)
    assert torch.equal(again, dbuf)


@pytest.mark.gpu
def test_group_norm_kernel_rejects_unsupported():
    t = torch.zeros(1, 4, 250, device=DEV)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        pkg.cabi.group_norm_tokens_(t, [4], torch.ones(1, 250, device=DEV), torch.zeros(1, 250, device=DEV), 25, 1e-5)
    t = torch.zeros(1, 4, 256, device=DEV)
    with pytest.raises(RuntimeError, match="divisible"):
        pkg.cabi.group_norm_tokens_(t, [4], torch.ones(1, 256, device=DEV), torch.zeros(1, 256, device=DEV), 24, 1e-5)


LP_SHAPES = [(12, 20), (6, 10), (3, 5), (2, 3)]  # token counts 240 / 60 (vectorised flatten kernel) and 15 / 6 (tile kernel)


@pytest.mark.gpu
def test_token_lpos_keep_bit_identical_to_flatten():
    gen = torch.Generator().manual_seed(7)
    b, c = 2, 256
    feats = [torch.randn(b, c, h, w, generator=gen).to(DEV) for h, w in LP_SHAPES]
    pos = [torch.randn(b, c, h, w, generator=gen).to(DEV) for h, w in LP_SHAPES]
    sizes = [h * w for h, w in LP_SHAPES]
    embeds = torch.randn(len(sizes), c, generator=gen).to(DEV)
    keep = (torch.rand(b, sum(sizes), generator=gen) > 0.3).float().to(DEV)
    feat_tok, lpos_want, x_want = pkg.cabi.flatten_tokens(feats, pos, embeds, keep)
    pos_tok = pkg.cabi.maps_to_tokens(pos)
    lpos, x = pkg.cabi.token_lpos_keep(feat_tok, pos_tok, embeds, keep, sizes)
    assert torch.equal(lpos, lpos_want) and torch.equal(x, x_want)
    lpos2, x2 = pkg.cabi.token_lpos_keep(feat_tok, pos_tok, embeds, keep, sizes, lpos=pos_tok)  # in place
    assert lpos2.data_ptr() == pos_tok.data_ptr() and torch.equal(lpos2, lpos_want) and torch.equal(x2, x_want)
    pos_tok = torch.randn(b, sum(sizes), c, generator=gen).to(DEV)
    _, lpos_want, x_want = pkg.cabi.flatten_tokens_pos(feats, pos_tok, embeds, keep)
    lpos, x = pkg.cabi.token_lpos_keep(feat_tok, pos_tok, embeds, keep, sizes)
    assert torch.equal(lpos, lpos_want) and torch.equal(x, x_want)


# ---- GPU: the module --------------------------------------------------------------------------------------------------
WIDTHS = {"resnet50": (512, 1024, 2048), "swin_l": (384, 768, 1536)}
SMALL_SHAPES = [(10, 14), (5, 7), (3, 4)]


def _mapper(cin):
    torch.manual_seed(5)
    return mcg.perturb_affine(pkg.ChannelMapper(list(cin), 256, len(cin) + 1)).eval()


def _inputs(cin, shapes, scale, channels_last, seed=3):
    g = torch.Generator().manual_seed(seed)
    xs = OrderedDict((str(i), torch.randn(2, c, h, w, generator=g) * scale) for i, (c, (h, w)) in enumerate(zip(cin, shapes)))
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    return xs, OrderedDict((k, v.to(DEV).contiguous(memory_format=fmt)) for k, v in xs.items())


def _ref64(m, xs):
    m64 = pkg.ChannelMapper(list(m.in_channels), 256, len(m.convs)).double()
    m64.load_state_dict(m.state_dict())
    with torch.no_grad():
        return [o.double() for o in _torch_chain(m64.cpu().eval(), OrderedDict((k, v.double()) for k, v in xs.items()))]


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last", [False, True])
def test_forward_tokens_vs_reference_fixture(channels_last):
    g = _golden()
    m = mcg.build(pkg.ChannelMapper).to(DEV)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    inputs = OrderedDict((k, v.to(DEV).contiguous(memory_format=fmt)) for k, v in mcg.inputs().items())
    with torch.no_grad():
        assert m.tokens_supported(inputs)
        tokens, shapes = m.forward_tokens(inputs)
        views = m(inputs)
    assert shapes == mcg.SHAPES + [(2, 3)]
    for i, v in enumerate(views):
        assert (v.cpu() - g[f"out{i}"]).abs().max() < 1e-4, i
    assert pkg.tokens_of(views) is not None and torch.equal(pkg.tokens_of(views), tokens)
    for v, t in zip(views, pkg.cabi.tokens_to_maps(tokens, shapes)):
        assert torch.equal(v.contiguous(), t)


@pytest.mark.gpu
@pytest.mark.parametrize("width", sorted(WIDTHS))
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("scale", [1e-3, 1e4])
def test_forward_tokens_vs_fp64(width, channels_last, scale):
    """ResNet-50 and Swin-L widths on small maps, NCHW and channels-last inputs, input scales 1e-3 and 1e4: within 1e-4 of the
    fp64 torch module on the O(1) GroupNorm outputs (the convolutions are 3xFP16, the GroupNorm fp32)"""
    cin = WIDTHS[width]
    m = _mapper(cin).to(DEV)
    xs, inputs = _inputs(cin, SMALL_SHAPES, scale, channels_last)
    with torch.no_grad():
        views = m(inputs)
        tokens, shapes = m.forward_tokens(inputs)
    assert pkg.tokens_of(views) is not None and torch.equal(pkg.tokens_of(views), tokens)
    want = _ref64(m, xs)
    err = max(float((v.cpu().double() - w).abs().max()) for v, w in zip(views, want))
    print(f"forward_tokens {width} channels_last={channels_last} scale={scale}: max err vs fp64 {err:.2e}")
    assert err <= 1e-4
    assert [tuple(v.shape) for v in views] == [tuple(w.shape) for w in want]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EXCLUDED) + ["training_with_grad"])
def test_excluded_configurations_fall_back_gpu(name):
    if name == "training_with_grad":
        m = mcg.build(pkg.ChannelMapper).train()
        inputs = mcg.inputs()
    else:
        m, inputs = _excluded(name)
    m = m.to(DEV)
    inputs = OrderedDict((k, v.to(DEV)) for k, v in inputs.items())
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        assert not m.tokens_supported(inputs)
        outs = m(inputs)
        with torch.no_grad():
            want = _torch_chain(m, inputs)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert pkg.tokens_of(outs) is None
    for a, b in zip(outs, want):
        assert torch.allclose(a, b, atol=1e-4, rtol=1e-4)
    if name == "training_with_grad":
        assert all(o.requires_grad for o in outs)


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last", [False, True])
def test_forward_tokens_graph_replay_and_launches(channels_last):
    m = mcg.build(pkg.ChannelMapper).to(DEV)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    inputs = OrderedDict((k, v.to(DEV).contiguous(memory_format=fmt)) for k, v in mcg.inputs().items())
    with torch.no_grad():
        eager, _ = m.forward_tokens(inputs)  # also builds the kernel weights outside the capture
        n0 = pkg.cabi.launch_count()
        eager2, _ = m.forward_tokens(inputs)
        want = m.launches_per_forward(0 if channels_last else 3)
        assert pkg.cabi.launch_count() - n0 == want == (11 if channels_last else 14)
        assert torch.equal(eager, eager2)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m.forward_tokens(inputs)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out, _ = m.forward_tokens(inputs)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)


@pytest.mark.gpu
def test_chained_extra_levels():
    """num_outs two above the inputs: the second extra conv reads the first extra level's normalised output"""
    cin = (128, 256)
    torch.manual_seed(9)
    m = mcg.perturb_affine(pkg.ChannelMapper(list(cin), 256, 4)).eval().to(DEV)
    xs, inputs = _inputs(cin, [(9, 13), (5, 7)], 1.0, False)
    with torch.no_grad():
        m(inputs)  # builds the kernel weights
        n0 = pkg.cabi.launch_count()
        views = m(inputs)
        assert pkg.cabi.launch_count() - n0 == m.launches_per_forward() == 2 + 8 + 6
    assert [tuple(v.shape[2:]) for v in views] == [(9, 13), (5, 7), (3, 4), (2, 2)]
    want = _ref64(m, xs)
    assert max(float((v.cpu().double() - w).abs().max()) for v, w in zip(views, want)) <= 1e-4


# ---- GPU: the transformer on token-backed features -------------------------------------------------------------------
MAP_CIN = (128, 256, 512)


def _transformer(with_decoder):
    geo = mg.HALF
    relu = nn.ReLU(inplace=True)
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(geo["embed_dim"], geo["d_ffn"], 0.0, geo["n_heads"], relu,
                                                                            4, 4, topk_sa=geo["topk_sa"]), geo["num_layers"],
                                         geo["max_num_embedding"])
    dec = neck = None
    if with_decoder:
        dec = pkg.SalienceTransformerDecoder(pkg.SalienceTransformerDecoderLayer(geo["embed_dim"], geo["d_ffn"], geo["n_heads"], 0.0,
                                                                                relu, 4, 4), geo["dec_layers"], geo["num_classes"])
        neck = pkg.RepVGGPluXNetwork([256] * 4, [256] * 4, groups=4, norm_layer=nn.BatchNorm2d, activation=nn.SiLU)
    tr = pkg.SalienceTransformer(enc, neck, dec, geo["num_classes"], 4, geo["num_proposals"], geo["level_filter_ratio"],
                                 geo["layer_filter_ratio"])
    own = tr.state_dict()
    sd = orc.deterministic_state_dict({k: v.shape for k, v in own.items() if not k.startswith("neck.") and
                                       not k.endswith("_filter_ratio")}, mg.HALF_SEED)
    if neck is not None:
        sd.update({"neck." + k: v for k, v in mng.neck_state_dict({k: v.shape for k, v in neck.state_dict().items()},
                                                                   mng.NECK_SEED).items()})
    tr.load_state_dict(sd, strict=False)
    tr.attach_position_embedding(pkg.PositionEmbeddingSine(128, temperature=10000, normalize=True, offset=-0.5))
    return tr.to(DEV).eval()


def _mapped_inputs():
    """backbone-like maps at the HALF level shapes through a ChannelMapper (3 inputs + 1 extra level = the 4 levels)"""
    feats, masks, pos = orc.synthetic_inputs(mg.image_sizes(True), (480, 640), 256, seed=mg.HALF_INPUT_SEED)
    shapes = [tuple(f.shape[2:]) for f in feats]
    torch.manual_seed(11)
    mapper = mcg.perturb_affine(pkg.ChannelMapper(list(MAP_CIN), 256, 4)).eval().to(DEV)
    _, inputs = _inputs(MAP_CIN, shapes[:3], 1.0, False, seed=12)
    return mapper, inputs, [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]


def _same(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("pos_form", ["maps", "attached"])
def test_encoder_on_token_backed_features(pos_form):
    tr = _transformer(False)
    mapper, inputs, masks, pos = _mapped_inputs()
    pos = pos if pos_form == "maps" else None
    with torch.no_grad():
        views = mapper(inputs)
        tokens = pkg.tokens_of(views)
        assert tokens is not None
        before = tokens.clone()
        mem, aux = tr.forward_encoder(views, masks, pos)
        mem_c, aux_c = tr.forward_encoder([v.contiguous() for v in views], masks, pos)
    torch.cuda.synchronize()
    assert torch.equal(tokens, before)  # the encoder never writes the mapper's buffer
    assert torch.equal(mem, mem_c)
    assert torch.equal(aux["selected_inds"], aux_c["selected_inds"]) and torch.equal(aux["raw_score"], aux_c["raw_score"])


@pytest.mark.gpu
@pytest.mark.parametrize("pos_form", ["maps", "attached"])
def test_full_transformer_on_token_backed_features(pos_form):
    tr = _transformer(True)
    mapper, inputs, masks, pos = _mapped_inputs()
    pos = pos if pos_form == "maps" else None
    with torch.no_grad():
        views = mapper(inputs)
        before = pkg.tokens_of(views).clone()
        got = tr(views, masks, pos, None, None, None)
        want = tr([v.contiguous() for v in views], masks, pos, None, None, None)
    torch.cuda.synchronize()
    assert len(got) == 5 and _same(list(got), list(want))
    assert torch.equal(pkg.tokens_of(views), before)


@pytest.mark.gpu
def test_mapper_and_encoder_in_one_cuda_graph():
    tr = _transformer(False)
    mapper, inputs, masks, pos = _mapped_inputs()
    with torch.no_grad():
        plan = tr.make_plan(masks)
        eager, _ = tr.forward_encoder(mapper(inputs), masks, pos, plan=plan)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            tr.forward_encoder(mapper(inputs), masks, pos, plan=plan)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            mem, _ = tr.forward_encoder(mapper(inputs), masks, pos, plan=plan)
        graph.replay()
        torch.cuda.synchronize()
        first = mem.clone()
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(first, eager) and torch.equal(mem, eager)
