"""What the backbone tests share (test_backbone.py, test_convnext_backbone.py, test_swin_backbone.py and
test_backbone_training.py): the golden fixtures, each backbone built on the fixtures' synthetic weights, padded image batches,
the float64 error harness, the backbone -> ChannelMapper -> encoder chain, and the checks every token-layout backbone passes
alike (weight loading; no host synchronisation, launch count, repeatability and CUDA-graph replay; golden outputs on the GPU),
each test file calling them with its backbone's constants."""
import contextlib
import copy
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch import nn

import salience_detr_b200 as pkg
from salience_detr_b200 import backbone as bbm
from salience_detr_b200 import convnext as cnm
from salience_detr_b200 import swin as swm
from salience_detr_b200 import synthetic
from conftest import GOLDEN
from oracle import make_golden as mg
from oracle import oracle as orc
from tools import make_backbone_golden as mbg
from tools import make_convnext_golden as mcg
from tools import make_swin_golden as msg

DEV = "cuda:0"
FBN = pkg.FrozenBatchNorm2d


def golden(name):
    """tests/golden/<name>.npz: tensors, and the parsed JSON of every key ending in _json"""
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    return {k: (json.loads(str(z[k])) if k.endswith("_json") else torch.from_numpy(z[k])) for k in z.files}


# ---- each backbone on the fixtures' synthetic weights (every key of the full network but the classifier's) ----------------
def resnet_weights(arch="resnet50"):
    net = bbm.ResNet(**pkg.ResNetBackbone.model_arch[arch], norm_layer=FBN)
    shapes = {k: list(v.shape) for k, v in net.state_dict().items() if not k.startswith("fc.")}
    return synthetic.resnet_weights(shapes, mbg.WEIGHT_SEED)


def convnext_weights(arch="conv_l"):
    net = cnm.ConvNeXt(**pkg.ConvNeXtBackbone.model_arch[arch])
    shapes = {k: list(v.shape) for k, v in net.state_dict().items() if not k.startswith("classifier.")}
    return synthetic.convnext_weights(shapes, mcg.WEIGHT_SEED)


def swin_weights(arch="swin_l"):
    net = swm.SwinTransformer(**pkg.SwinTransformerBackbone.model_arch[arch])
    return synthetic.swin_weights({k: v for k, v in net.state_dict().items() if not k.startswith(("norm.", "head."))},
                                  msg.WEIGHT_SEED)


def resnet_backbone(arch="resnet50", return_indices=(1, 2, 3), freeze_indices=(0,), **kw):
    return pkg.ResNetBackbone(arch, weights=resnet_weights(arch), return_indices=return_indices, freeze_indices=freeze_indices,
                              norm_layer=kw.pop("norm_layer", FBN), **kw)


_WEIGHTS = {}


def convnext_backbone(arch="conv_l", return_indices=(1, 2, 3), freeze_indices=(0,), **kw):
    if arch not in _WEIGHTS:
        _WEIGHTS[arch] = convnext_weights(arch)
    return pkg.ConvNeXtBackbone(arch, weights=_WEIGHTS[arch], return_indices=return_indices, freeze_indices=freeze_indices,
                                **kw).eval()


def swin_backbone(arch="swin_l", return_indices=(1, 2, 3), freeze_indices=(0,), **kw):
    if arch not in _WEIGHTS:
        _WEIGHTS[arch] = swin_weights(arch)
    return pkg.SwinTransformerBackbone(arch, weights=_WEIGHTS[arch], return_indices=return_indices,
                                       freeze_indices=freeze_indices, **kw).eval()


# ---- inputs and errors ------------------------------------------------------------------------------------------------------
def padded_images(b, H, W, gen, step=(37, 61)):
    """b images in an (H, W) batch, image i of (H - step[0] i, W - step[1] i) pixels (at least 1) and zero padding
    (image_list_from_tensors' layout)"""
    x = torch.zeros(b, 3, H, W)
    for i in range(b):
        h, w = max(1, H - step[0] * i), max(1, W - step[1] * i)
        x[i, :, :h, :w] = torch.randn(3, h, w, generator=gen)
    return x


def resnet_images(b, H, W, gen):
    """padded_images with the ResNet tests' step: image i of (H - 3 i, W - 5 i) pixels"""
    return padded_images(b, H, W, gen, (3, 5))


def rel_err(got, ref):
    return float((got.double() - ref).abs().max()) / float(ref.abs().max())


@contextlib.contextmanager
def tf32(enabled):
    """TF32 on or off for both cuDNN and cuBLAS, restored on exit"""
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = enabled
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


def errors(m, x):
    """per output: (token path, torch fp32, torch TF32) max |err| / max |ref| against forward() in float64, and the token
    path's outputs"""
    m64 = copy.deepcopy(m).double()
    with torch.no_grad():
        ref = m64(x.double())
        del m64
        tok = m(x)
        with tf32(False):
            fp32 = m.forward_torch(x)
        with tf32(True):
            t32 = m.forward_torch(x)
    return {k: (rel_err(tok[k], ref[k]), rel_err(fp32[k], ref[k]), rel_err(t32[k], ref[k])) for k in ref}, tok


def graph_replay(fn):
    """fn() once on a side stream, then captured in a CUDA graph and replayed: (the graph, its outputs)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    graph.replay()
    torch.cuda.synchronize()
    return graph, out


# ---- backbone -> ChannelMapper -> encoder ------------------------------------------------------------------------------------
def encoder():
    geo = mg.HALF
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(geo["embed_dim"], geo["d_ffn"], 0.0, geo["n_heads"],
                                                                            nn.ReLU(inplace=True), 4, 4, topk_sa=geo["topk_sa"]),
                                         geo["num_layers"], geo["max_num_embedding"])
    tr = pkg.SalienceTransformer(enc, None, None, geo["num_classes"], 4, geo["num_proposals"], geo["level_filter_ratio"],
                                 geo["layer_filter_ratio"])
    sd = orc.deterministic_state_dict({k: v.shape for k, v in tr.state_dict().items() if not k.endswith("_filter_ratio")},
                                      mg.HALF_SEED)
    tr.load_state_dict(sd, strict=False)
    return tr.to(DEV).eval()


def mapper_chain(bb):
    """Images at the half-width encoder's sizes -> bb (on the GPU) -> ChannelMapper(bb.num_channels) -> forward_encoder, after
    checking that the mapper takes bb's maps with zero transposes.  -> namespace of x, masks, pos, mapper, tr (the encoder),
    plan, mapped (the mapper's tokens), mem (the encoder memory), ref_feats (bb's maps in float64) and ref_mapped (the mapper's
    tokens of those)."""
    sizes = mg.image_sizes(True)
    _, masks, pos = orc.synthetic_inputs(sizes, (480, 640), 256, seed=mg.HALF_INPUT_SEED)
    masks, pos = [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]
    gen = torch.Generator().manual_seed(21)
    x = torch.zeros(len(sizes), 3, 480, 640)
    for i, (h, w) in enumerate(sizes):
        x[i, :, :h, :w] = torch.randn(3, h, w, generator=gen)
    x = x.to(DEV)
    torch.manual_seed(11)
    mapper = pkg.ChannelMapper(bb.num_channels, 256, 4).eval().to(DEV)
    tr = encoder()
    with torch.no_grad():
        feats = bb(x)
        mapper(feats)  # builds the mapper's kernel weights
        assert [tuple(v.shape[2:]) for v in feats.values()] == [tuple(m.shape[1:]) for m in masks[:3]]
        n0 = pkg.cabi.launch_count()
        mapped, _ = mapper.forward_tokens(feats)
        assert pkg.cabi.launch_count() - n0 == mapper.launches_per_forward(0)  # no transposes
        plan = tr.make_plan(masks)
        mem = tr.forward_encoder(mapper(feats), masks, pos, plan=plan)[0]
        ref_feats = copy.deepcopy(bb).double()(x.double())
        ref_mapped = mapper.forward_tokens({k: v.float().contiguous(memory_format=torch.channels_last)
                                            for k, v in ref_feats.items()})[0]
    return SimpleNamespace(x=x, masks=masks, pos=pos, mapper=mapper, tr=tr, plan=plan, mapped=mapped, mem=mem,
                           ref_feats=ref_feats, ref_mapped=ref_mapped)


def chain_graph_matches_eager(bb, c):
    """the whole chain captured in one CUDA graph gives the eager encoder memory bit for bit"""
    with torch.no_grad():
        _, out = graph_replay(lambda: c.tr.forward_encoder(c.mapper(bb(c.x)), c.masks, c.pos, plan=c.plan)[0])
    return torch.equal(out, c.mem)


# ---- the checks every token-layout backbone passes alike --------------------------------------------------------------------
def check_weight_loading(tmp_path, cls, arch, weights, kw, classifier, drop, resize, url, bad_arch):
    """``cls(arch, weights=...)`` with ``kw`` takes the synthetic ``weights(arch)`` as a state dict, with the ``classifier``
    keys of a full checkpoint added, under "model" and from a local path, all to the same state; it refuses a state dict
    without the key ``drop`` or with an extra key or a wrong-sized ``resize``, the download ``url`` and the arch ``bad_arch``"""
    sd = weights(arch)
    full = dict(sd, **classifier)
    want = cls(arch, weights=sd, return_indices=(1, 2, 3), **kw).state_dict()
    assert all(torch.equal(want[k], sd[k]) for k in want)
    for w in (sd, full, {"model": full}):
        m = cls(arch, weights=w, return_indices=(1, 2, 3), **kw)
        assert all(torch.equal(m.state_dict()[k], v) for k, v in want.items())
    path = tmp_path / f"{arch}.pth"
    torch.save({"model": full}, path)
    m = cls(arch, weights=str(path), return_indices=(1, 2, 3), **kw)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in want.items())
    with pytest.raises(RuntimeError, match="missing"):
        cls(arch, weights={k: v for k, v in sd.items() if k != drop}, **kw)
    with pytest.raises(RuntimeError, match="unexpected"):
        cls(arch, weights=dict(sd, extra=torch.zeros(1)), **kw)
    with pytest.raises(RuntimeError, match="size mismatch"):
        cls(arch, weights=dict(sd, **{resize: torch.zeros(3)}), **kw)
    with pytest.raises(RuntimeError, match="downloading weights is not supported"):
        cls(arch, weights=url)
    with pytest.raises(ValueError, match="architecture"):
        cls(bad_arch)


def check_no_sync_graph_replay_repeatability_and_launches(m, x, launches):
    """m(x) on the GPU without a host synchronisation in ``launches`` library launches (= m.launches_per_forward()), the same
    bits again and from a CUDA-graph replay"""
    with torch.no_grad():
        eager = m(x)  # also builds the kernel weights outside the capture
        eager = {k: v.clone() for k, v in eager.items()}
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            n0 = pkg.cabi.launch_count()
            again = m(x)
            assert pkg.cabi.launch_count() - n0 == m.launches_per_forward() == launches
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert all(torch.equal(eager[k], again[k]) for k in eager)
        _, out = graph_replay(lambda: m(x))
    assert all(torch.equal(out[k], eager[k]) for k in eager)


def check_golden_outputs_on_gpu(m, fixture):
    """m on the GPU takes the token path on the fixture's image and gives its outputs within 1e-5 of their largest value"""
    g = golden(fixture)
    m = m.to(DEV)
    with torch.no_grad():
        assert m.tokens_supported(g["image"].to(DEV))
        outs = m(g["image"].to(DEV))
    for k, v in outs.items():
        want = g[f"out.{k}"]
        assert float((v.cpu() - want).abs().max()) <= 1e-5 * float(want.abs().max()), k
