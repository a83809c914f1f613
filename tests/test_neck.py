"""RepVGG-PluX neck (neck.py): the torch mirror against the UNMODIFIED reference (tests/golden/neck_repnet.npz and
transformer_neck.npz, made by tools/make_neck_golden.py), the eval-weight folding and nearest-index rule on the CPU, and the
token-layout kernels (sdetr_conv2d_f16x3, sdetr_context_gate, sdetr_upsample_nearest_concat) and forward_tokens on the GPU."""
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import salience_detr_b200 as pkg
from conftest import GOLDEN
from oracle import make_golden as mg
from oracle import oracle as orc
from tools import make_neck_golden as mng

DEV = "cuda:0"
C, G = mng.CHANNELS, mng.GROUPS


def _golden(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return {k: (str(z[k]) if z[k].dtype.kind in "US" else torch.from_numpy(z[k])) for k in z.files}


def _net(dtype=torch.float32):
    g = _golden("neck_repnet.npz")
    net = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=G, norm_layer=torch.nn.BatchNorm2d, activation=torch.nn.SiLU)
    shapes = json.loads(g["shapes_json"])
    net.load_state_dict(mng.neck_state_dict(shapes, mng.NECK_SEED), strict=True)
    return net.to(dtype).eval(), g


def _rows(tok, idx):
    return torch.gather(tok, 1, idx[..., None].expand(-1, -1, tok.shape[2]))


def _folded_forward(net, feats):
    """forward_tokens' dataflow written with torch ops on the folded weights (NCHW), for the CPU check of the folding"""
    def conv(x, wb, stride=1, groups=1):
        w, b = wb
        return F.silu(F.conv2d(x, w, b, stride, w.shape[-1] // 2, groups=groups))

    def gate(se, y, x):
        n, c, h, w = y.shape
        p = F.conv2d(y, se.conv_mask.weight, se.conv_mask.bias).view(n, h * w).softmax(-1)
        ctx = torch.einsum("ncp,np->nc", y.view(n, c, h * w), p)
        hid = F.relu(ctx @ se.se_module[0].weight.view(-1, c).T)
        return torch.sigmoid(hid @ se.se_module[2].weight.view(c, -1).T)[:, :, None, None] * y + x

    def csp(layer, x):
        proj = conv(x, pkg.neck.fold_csp_projection(layer))
        h, r = proj.chunk(2, 1)
        for blk in layer.bottlenecks:
            h = gate(blk.se_module, conv(h, pkg.neck.fold_repvgg(blk), groups=G), h)
        return h + r

    lat, tops, x = {}, {}, feats
    hi = x[-1]
    for idx in range(len(x) - 1, 0, -1):
        lat[idx] = conv(hi, pkg.neck.fold_conv_norm(net.lateral_convs[idx - 1]))
        up = F.interpolate(lat[idx], size=x[idx - 1].shape[-2:], mode="nearest")
        hi = tops[idx - 1] = csp(net.layer_blocks[idx - 1], torch.cat([up, x[idx - 1]], 1))
    outs = [tops[0]]
    for idx in range(len(x) - 1):
        d = conv(outs[-1], pkg.neck.fold_conv_norm(net.downsample_blocks[idx]), stride=2)
        outs.append(csp(net.pan_blocks[idx], torch.cat([d, lat[idx + 1]], 1)))
    return outs


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_state_dict_matches_reference_keys():
    net, g = _net()
    want = json.loads(g["shapes_json"])
    assert {k: list(v.shape) for k, v in net.state_dict().items()} == want
    assert len(want) > 390 and any(k.endswith("num_batches_tracked") for k in want)
    blk = pkg.RepVggPluXBlock(C, C, activation_layer=torch.nn.SiLU, groups=G, alpha=True)
    bwant = json.loads(g["block_shapes_json"])
    assert {k: list(v.shape) for k, v in blk.state_dict().items()} == bwant and "alpha" in bwant
    blk.load_state_dict(mng.neck_state_dict(bwant, mng.BLOCK_SEED), strict=True)


def test_reference_checkpoint_has_no_unexpected_neck_keys():
    net, g = _net()
    shapes = json.loads(g["shapes_json"])
    ckpt = {"model": {"transformer.neck." + k: v for k, v in mng.neck_state_dict(shapes, 5).items()}}
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(C, 64, 0.0, 8), 1, 40)
    tr = pkg.SalienceTransformer(enc, pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=G), None)
    res = pkg.load_reference_checkpoint(tr, ckpt)
    assert res["unexpected"] == [] and res["mismatched"] == []
    assert not any(k.startswith("neck.") for k in res["missing"])
    assert torch.equal(tr.neck.pan_blocks[1].bottlenecks[2].conv1[1].running_var, ckpt["model"][
        "transformer.neck.pan_blocks.1.bottlenecks.2.conv1.1.running_var"])


def test_folded_weights_reproduce_eval_module_fp64():
    """BatchNorm folding, RepVGG 3x3 + alpha 1x1 merge (alpha=True block) and the CSP conv1 || conv2 concatenation, in fp64:
    round-off agreement with the unfolded eval modules, and the whole folded dataflow against forward()."""
    torch.manual_seed(0)
    blk = pkg.RepVggPluXBlock(C, C, activation_layer=torch.nn.SiLU, groups=G, alpha=True)
    blk.load_state_dict(mng.neck_state_dict({k: v.shape for k, v in blk.state_dict().items()}, mng.BLOCK_SEED))
    blk = blk.double().eval()
    assert abs(float(blk.alpha.detach()) - 1.0) > 0.01
    x = torch.randn(2, C, 9, 11, dtype=torch.float64)
    w, b = pkg.neck.fold_repvgg(blk)
    with torch.no_grad():
        want = blk.conv1(x) + blk.alpha * blk.conv2(x)
    assert (F.conv2d(x, w, b, 1, 1, groups=G) - want).abs().max() < 1e-12 * max(1.0, float(want.abs().max()))
    net, _ = _net(torch.float64)
    xs = torch.randn(2, 2 * C, 7, 5, dtype=torch.float64)
    with torch.no_grad():
        lay = net.layer_blocks[0]
        want = torch.cat([lay.conv1(xs), lay.conv2(xs)], 1)
        got = F.silu(F.conv2d(xs, *pkg.neck.fold_csp_projection(lay)))
        assert (got - want).abs().max() < 1e-12
        feats = [t.double() for t in mng.neck_inputs()]
        ref = list(net(OrderedDict(enumerate(feats))).values())
        fold = _folded_forward(net, feats)
    for a, r in zip(fold, ref):
        assert (a - r).abs().max() < 1e-10 * max(1.0, float(r.abs().max()))


@pytest.mark.parametrize("src,dst", [((13, 21), (25, 42)), ((25, 42), (50, 84)), ((8, 10), (15, 20)), ((7, 11), (20, 30))])
def test_nearest_index_matches_interpolate(src, dst):
    x = torch.arange(src[0] * src[1], dtype=torch.float64).view(1, 1, *src)
    want = F.interpolate(x, size=dst, mode="nearest")[0, 0]
    iy, ix = pkg.neck.nearest_index(src[0], dst[0]), pkg.neck.nearest_index(src[1], dst[1])
    assert torch.equal(want, x[0, 0][iy][:, ix])


def test_torch_forward_matches_reference_eval_and_train():
    net, g = _net()
    feats = mng.neck_inputs()
    with torch.no_grad():
        ev = mng.tokens(list(net(OrderedDict(enumerate(feats))).values()))
        assert (_rows(ev, g["rows_index"]) - g["eval_rows"]).abs().max() < 1e-4 * max(1.0, float(g["eval_absmax"]))
        tr = mng.tokens(list(net.train()(OrderedDict(enumerate(feats))).values()))
    assert (_rows(tr, g["rows_index"]) - g["train_rows"]).abs().max() < 1e-4 * max(1.0, float(g["train_rows"].abs().max()))
    sd = net.state_dict()
    for name in mng.TRAIN_STATS:
        for s in ("running_mean", "running_var"):
            assert (sd[f"{name}.{s}"] - g[f"train.{name}.{s}"]).abs().max() < 1e-5, (name, s)
        assert int(sd[f"{name}.num_batches_tracked"]) == int(g[f"train.{name}.num_batches_tracked"]) == 8
    blk = pkg.RepVggPluXBlock(C, C, activation_layer=torch.nn.SiLU, groups=G, alpha=True)
    blk.load_state_dict(mng.neck_state_dict(json.loads(g["block_shapes_json"]), mng.BLOCK_SEED), strict=True)
    with torch.no_grad():
        out = blk.eval()(mng.block_input())
    assert (out.reshape(-1)[g["block_out_idx"]] - g["block_out"]).abs().max() < 1e-4 * max(1.0, float(g["block_out_absmax"]))
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(net)
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in sync.modules())


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _level_slice(b, shapes, lvl, c, gen, scale=1.0):
    """a (b, H*W, c) level slice of a (b, Nv, c) token tensor (image pitch != H*W*c) and the tensor"""
    sizes = [h * w for h, w in shapes]
    t = (torch.randn(b, sum(sizes), c, generator=gen) * scale).to(DEV)
    s = sum(sizes[:lvl])
    return t[:, s:s + sizes[lvl]], t


CONV_KINDS = {"3x3_s1_g4": (3, 1, G, C, C), "3x3_s2_g1": (3, 2, 1, C, C), "1x1_s1_g1": (1, 1, 1, 2 * C, 2 * C)}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(CONV_KINDS))
@pytest.mark.parametrize("b", [1, 2])
def test_conv_kernel_vs_fp64(kind, b):
    """sdetr_conv2d_f16x3 on level slices, into level slices, against fp64 F.conv2d.  Tolerance: the 3xFP16 product keeps ~22
    significand bits per operand and every 64-wide k-block is added in fp32, so |err| <= 2^-17 * (|x| conv |W|) (fp64), plus
    the SiLU, whose slope is below 1.1 -- far below a TF32 or fp16 convolution's error (~2^-11 of the same sum)."""
    k, stride, groups, cin, cout = CONV_KINDS[kind]
    gen = torch.Generator().manual_seed(hash(kind) % 1000 + b)
    maps = [(1, 1), (1, 7), (13, 21), (25, 42), (100, 168)]
    w = torch.randn(cout, cin // groups, k, k, generator=gen) / (cin // groups * k * k) ** 0.5
    bias = torch.randn(cout, generator=gen) * 0.1
    w_hi, w_lo, w_scale = pkg.cabi.split_f16_pair_dev(w.permute(0, 2, 3, 1).contiguous().to(DEV))
    for i, (h, wd) in enumerate(maps):
        for scale in (1e-3, 1.0, 1e4):
            x, base = _level_slice(b, [(3, 5), (h, wd), (2, 2)], 1, cin, gen, scale)
            ho, wo = (h + 2 * (k // 2) - k) // stride + 1, (wd + 2 * (k // 2) - k) // stride + 1
            _, obase = _level_slice(b, [(4, 4), (ho, wo)], 1, cout, gen)
            out = obase[:, 16:]
            x64 = x.double().transpose(1, 2).reshape(b, cin, h, wd).cpu()
            ref = F.conv2d(x64, w.double(), bias.double() * scale, stride, k // 2, groups=groups)
            bnd = F.conv2d(x64.abs(), w.double().abs(), None, stride, k // 2, groups=groups) + (bias.double() * scale).abs().view(1, -1, 1, 1)
            for act in (0, pkg.cabi.ACT_SILU):
                sentinel = obase[:, :16].clone()
                pkg.cabi.conv2d_f16x3(x, (h, wd), pkg.cabi.pow2_scale(base, 12), w_hi, w_lo, w_scale, (bias * scale).to(DEV),
                                      groups, k, stride, act, out=out)
                got = out.cpu().double().transpose(1, 2).reshape(b, cout, ho, wo)
                want = F.silu(ref) if act else ref
                err = (got - want).abs()
                assert bool((err <= 2.0 ** -17 * 1.1 * bnd + 1e-30).all()), (kind, b, h, wd, scale, act, float(err.max()))
                assert torch.equal(obase[:, :16], sentinel)  # nothing outside the output slice is written


@pytest.mark.gpu
def test_conv_kernel_rejects_unsupported_shapes():
    x = torch.zeros(1, 4, 96, device=DEV)
    hi = torch.zeros(96, 1, 1, 96, device=DEV, dtype=torch.float16)
    s = torch.ones(1, device=DEV)
    with pytest.raises(RuntimeError, match="multiples of 64"):
        pkg.cabi.conv2d_f16x3(x, (2, 2), s, hi, hi, s, None, 1, 1, 1, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [1, 300, 16800])
def test_context_gate_vs_fp64(hw):
    """one image of 1 pixel, a pixel count that does not divide the 128-pixel chunk, and the largest config-2 level; logits
    spanning +-60; fp32 sums in a fixed order: within 2e-5 of fp64 (relative to the operands' magnitude) and bit-identical
    from run to run, with and without the second addend."""
    gen = torch.Generator().manual_seed(hw)
    b, r = 2, C // 16
    y, _ = _level_slice(b, [(1, 3), (1, hw)], 1, C, gen)
    x = torch.randn(b, hw, C, generator=gen).to(DEV)
    z = torch.randn(b, hw, C, generator=gen).to(DEV)
    w_mask = torch.randn(C, generator=gen) * 2.0   # logits ~ N(0, 32^2): softmax over a wide range
    b_mask = torch.randn(1, generator=gen)
    w1, w2 = torch.randn(r, C, generator=gen) / C ** 0.5, torch.randn(C, r, generator=gen) / r ** 0.5
    y64, x64, z64 = y.double().cpu(), x.double().cpu(), z.double().cpu()
    logit = y64 @ w_mask.double() + b_mask.double()
    assert logit.max() - logit.min() > 60 or hw == 1
    ctx = torch.einsum("npc,np->nc", y64, logit.softmax(1))
    gate = torch.sigmoid(F.relu(ctx @ w1.double().T) @ w2.double().T)
    args = [t.to(DEV) for t in (w_mask, b_mask, w1, w2)]
    for zz, zz64 in ((None, 0.0), (z, z64)):
        want = gate[:, None] * y64 + x64 + zz64
        got = pkg.cabi.context_gate(y, x, *args, z=zz)
        again = pkg.cabi.context_gate(y, x, *args, z=zz)
        assert torch.equal(got, again)
        assert (got.cpu().double() - want).abs().max() < 2e-5 * (1.0 + float(y64.abs().max()))


@pytest.mark.gpu
def test_upsample_concat_exact():
    gen = torch.Generator().manual_seed(3)
    for src, dst in [((13, 21), (25, 42)), ((7, 11), (20, 30)), ((1, 1), (3, 2))]:
        hi, _ = _level_slice(2, [(2, 2), src], 1, C, gen)
        lo, _ = _level_slice(2, [dst, (1, 1)], 0, C, gen)
        got = pkg.cabi.upsample_nearest_concat(hi, src, lo, dst)
        up = F.interpolate(hi.transpose(1, 2).reshape(2, C, *src), size=dst, mode="nearest").flatten(2).transpose(1, 2)
        assert torch.equal(got, torch.cat([up, lo], 2))


def _tokens_inputs():
    return mng.tokens(mng.neck_inputs()).to(DEV).contiguous()


@pytest.mark.gpu
def test_forward_tokens_vs_reference_and_fp64():
    net, g = _net()
    net = net.to(DEV)
    mem = _tokens_inputs()
    with torch.no_grad():
        assert net.tokens_supported(mem, mng.HALF_SHAPES)
        got = net.forward_tokens(mem, mng.HALF_SHAPES)
        n64 = _net(torch.float64)[0]
        ref64 = mng.tokens(list(n64(OrderedDict(enumerate(t.double() for t in mng.neck_inputs()))).values()))
    amax = max(1.0, float(g["eval_absmax"]))
    assert (_rows(got, g["rows_index"].to(DEV)).cpu() - g["eval_rows"]).abs().max() < 1e-4 * amax
    assert (got.cpu().double() - ref64).abs().max() < 5e-5 * amax
    net.train()
    assert not net.tokens_supported(mem, mng.HALF_SHAPES)  # training: BatchNorm batch statistics -> forward()


@pytest.mark.gpu
def test_forward_tokens_graph_replay_and_launches():
    net, _ = _net()
    net = net.to(DEV)
    mem = _tokens_inputs()
    with torch.no_grad():
        eager = net.forward_tokens(mem, mng.HALF_SHAPES)  # also folds the weights outside the capture
        n0 = pkg.cabi.launch_count()
        eager2 = net.forward_tokens(mem, mng.HALF_SHAPES)
        assert pkg.cabi.launch_count() - n0 == net.launches_per_forward(4, 3) == 117
        assert torch.equal(eager, eager2)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            net.forward_tokens(mem, mng.HALF_SHAPES)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = net.forward_tokens(mem, mng.HALF_SHAPES)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, eager)


@pytest.mark.gpu
def test_transformer_with_neck_vs_reference():
    """SalienceTransformer(encoder, RepVGGPluXNetwork, decoder) with the fixture's whole state dict loaded (the only missing keys:
    the *_filter_ratio buffers): the decoder's `value` rows within the neck hand-off bound, and the 5-tuple checked as in
    test_full_transformer_forward_vs_reference."""
    g = _golden("transformer_neck.npz")
    geo = mg.HALF
    relu = torch.nn.ReLU(inplace=True)
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(geo["embed_dim"], geo["d_ffn"], 0.0, geo["n_heads"], relu,
                                                                            4, 4, topk_sa=geo["topk_sa"]), geo["num_layers"],
                                         geo["max_num_embedding"])
    dec = pkg.SalienceTransformerDecoder(pkg.SalienceTransformerDecoderLayer(geo["embed_dim"], geo["d_ffn"], geo["n_heads"], 0.0, relu,
                                                                            4, 4), geo["dec_layers"], geo["num_classes"])
    neck = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=G, norm_layer=torch.nn.BatchNorm2d, activation=torch.nn.SiLU)
    ours = pkg.SalienceTransformer(enc, neck, dec, geo["num_classes"], 4, geo["num_proposals"], geo["level_filter_ratio"],
                                   geo["layer_filter_ratio"])
    sd = orc.deterministic_state_dict(json.loads(g["shapes_json"]), mg.HALF_SEED)
    sd.update({"neck." + k: v for k, v in mng.neck_state_dict({k: v.shape for k, v in neck.state_dict().items()}, mng.NECK_SEED).items()})
    res = ours.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and all(k.endswith("_filter_ratio") for k in res.missing_keys)
    ours = ours.to(DEV).eval()
    feats, masks, pos = orc.synthetic_inputs(mg.image_sizes(False), (480, 640), geo["embed_dim"], seed=mg.HALF_INPUT_SEED)
    feats, masks, pos = [f.to(DEV) for f in feats], [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]
    cap = {}
    dec_fwd = ours.decoder.forward

    def spy(**kw):
        cap["value"] = kw["value"]
        return dec_fwd(**kw)

    ours.decoder.forward = spy
    mode = pkg.gemm.MODE
    try:
        with torch.no_grad():
            pkg.gemm.MODE = "fp32"
            n0 = pkg.cabi.launch_count()
            got = ours(feats, masks, pos, None, None, None)
            assert pkg.cabi.launch_count() - n0 > ours.neck.launches_per_forward(4, 3)
    finally:
        pkg.gemm.MODE = mode
        del ours.decoder.forward
    v = _rows(cap["value"], g["value_rows_index"].to(DEV)).cpu()
    assert (v - g["value_rows"]).abs().max() < 2e-3 * max(1.0, float(g["value_absmax"]))
    want = [g[f"full{i}"] for i in range(4)] + [[g[f"full_score{i}"] for i in range(len([k for k in g if k.startswith("full_score")]))]]
    got = [t.cpu() for t in got[:4]] + [[t.cpu() for t in got[4]]]
    assert got[0].shape == want[0].shape and got[1].shape == want[1].shape and len(got[4]) == len(want[4])
    for a, w in zip(got[4], want[4]):
        assert a.shape == w.shape and (a - w).abs().max() < 1e-4
    same = (got[3] - want[3]).abs().amax(-1) < 1e-4
    assert same.float().mean() > 0.9
    assert (got[2] - want[2]).abs().amax(-1)[same].max() < 1e-3
    if bool(same.all()):
        assert (got[0] - want[0]).abs().max() < 2e-3 and (got[1] - want[1]).abs().max() < 2e-4
