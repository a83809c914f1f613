"""Decoder half (SURVEY.md 8(f)-1) against the UNMODIFIED reference modules: two-stage proposal selection
(salience_transformer.py:194-212, 249-295) and the decoder (:498-674) with 4-d reference boxes through the fused sampling kernel.
What the reference computes is stored in tests/golden/{nms_topk,decoder_half_even,decoder_half_ragged}.npz (oracle/make_golden.py
runs the original project on the same deterministic weights -- oracle.deterministic_state_dict -- and seeded inputs)."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import make_golden as mg
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GEO = mg.HALF


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


@pytest.fixture(autouse=True)
def _fp32(pkg):
    prev, mode = torch.backends.cuda.matmul.allow_tf32, pkg.gemm.MODE
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev
    pkg.gemm.MODE = mode


def _golden(ragged):
    z = np.load(os.path.join(GOLDEN, "decoder_half_%s.npz" % ("ragged" if ragged else "even")), allow_pickle=False)
    return {k: torch.from_numpy(z[k]) for k in z.files if k != "shapes_json"}, json.loads(str(z["shapes_json"]))


def _ours(pkg, shapes):
    """this package's transformer with a GEO["dec_layers"]-layer decoder and the fixture's weights (every reference key)"""
    relu = torch.nn.ReLU(inplace=True)
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(GEO["embed_dim"], GEO["d_ffn"], 0.0, GEO["n_heads"], relu,
                                                                            4, 4, topk_sa=GEO["topk_sa"]), GEO["num_layers"],
                                         GEO["max_num_embedding"])
    dec = pkg.SalienceTransformerDecoder(pkg.SalienceTransformerDecoderLayer(GEO["embed_dim"], GEO["d_ffn"], GEO["n_heads"], 0.0, relu,
                                                                            4, 4), GEO["dec_layers"], GEO["num_classes"])
    ours = pkg.SalienceTransformer(enc, None, dec, GEO["num_classes"], 4, GEO["num_proposals"], GEO["level_filter_ratio"],
                                   GEO["layer_filter_ratio"])
    res = ours.load_state_dict(orc.deterministic_state_dict(shapes, mg.HALF_SEED), strict=False)
    assert not res.unexpected_keys and all(k.endswith("_filter_ratio") for k in res.missing_keys)
    return ours.to(DEV).eval()


def _inputs(ragged):
    feats, masks, pos = orc.synthetic_inputs(mg.image_sizes(ragged), (480, 640), GEO["embed_dim"], seed=mg.HALF_INPUT_SEED)
    return [f.to(DEV) for f in feats], [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]


def test_nms_on_topk_index_matches_torchvision(pkg):
    """sdetr_nms_topk_index vs the reference's own nms_on_topk_index (torchvision.ops.batched_nms), index for index: its
    kept lists for the same seeded candidates are stored in tests/golden/nms_topk.npz (oracle/make_golden.py)."""
    z = np.load(os.path.join(GOLDEN, "nms_topk.npz"))
    g = torch.Generator().manual_seed(0)
    for i, (shapes, k) in enumerate([([(60, 80), (30, 40), (15, 20), (8, 10)], 1200),
                                     ([(100, 168), (50, 84), (25, 42), (13, 21)], 3600), ([(20, 20), (10, 10)], 450)]):
        st = torch.tensor(shapes, device=DEV)
        lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
        nv = int(st.prod(1).sum())
        scores = torch.rand(2, nv, generator=g).to(DEV)  # distinct with probability 1: the order is unambiguous
        topk_scores, topk_index = torch.topk(scores, k, dim=1)
        want = torch.from_numpy(z[f"kept{i}"]).to(DEV)
        kept, count, flag = pkg.cabi.nms_topk_index(topk_index.contiguous(), shapes, 0.3)
        n = want.shape[1]
        assert int(count.min()) >= n and torch.equal(kept[:, :n], want)
        for b in range(2):  # the verdicts are a valid greedy NMS: no two kept 4-neighbours, every suppressed one has a kept better neighbour
            assert int(flag[b].sum()) == int(count[b])
    ours = pkg.SalienceTransformer(pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(64, 64, 0.0, 2), 1, 40), None, None,
                                   two_stage_num_proposals=900)
    assert torch.equal(ours.nms_on_topk_index(topk_scores, topk_index, st, lsi), want)


@pytest.mark.parametrize("ragged", [False, True])
def test_decoder_on_reference_inputs(pkg, ragged):
    """The decoder alone on identical inputs on both sides (the reference filter's padding mask, valid ratios and proposal boxes,
    seeded memory, the learned target queries): class logits and boxes of every layer within 1e-3 / 1e-4 of the reference
    decoder's, in the strict fp32-GEMM mode and in the default tensor-core mode; then with denoising queries and their attention
    mask (salience_transformer.py:218-221)."""
    g, shapes = _golden(ragged)
    ours = _ours(pkg, shapes)
    b = g["reference_points"].shape[0]
    kw = dict(query=ours.tgt_embed.weight.expand(b, -1, -1),
              value=orc.seeded_memory((b, int(g["key_padding_mask"].shape[1]), GEO["embed_dim"]), mg.HALF_VALUE_SEED).to(DEV),
              key_padding_mask=g["key_padding_mask"].to(DEV), reference_points=g["reference_points"].to(DEV),
              spatial_shapes=g["spatial_shapes"].to(DEV), level_start_index=g["level_start_index"].to(DEV),
              valid_ratios=g["valid_ratios"].to(DEV), attn_mask=None)
    for mode in ("fp32", "auto"):
        pkg.gemm.MODE = mode
        n0 = pkg.cabi.launch_count()
        with torch.no_grad():
            cls, box = ours.decoder(**kw)
        assert pkg.cabi.launch_count() > n0 + 3 * GEO["dec_layers"]
        assert cls.shape == g["dec_cls"].shape and box.shape == g["dec_box"].shape
        assert (cls.cpu() - g["dec_cls"]).abs().max() < 1e-3, mode
        assert (box.cpu() - g["dec_box"]).abs().max() < 1e-4, mode
    dn_q, dn_b, mask = orc.denoising_queries(b, kw["query"].shape[1], GEO["embed_dim"])
    kw2 = dict(kw, query=torch.cat([dn_q.to(DEV), kw["query"]], 1), reference_points=torch.cat([dn_b.to(DEV), kw["reference_points"]], 1),
               attn_mask=mask.to(DEV))
    with torch.no_grad():
        pkg.gemm.MODE = "auto"
        g2 = ours.decoder(**kw2)
    assert (g2[0].cpu() - g["dn_cls"]).abs().max() < 1e-3 and (g2[1].cpu() - g["dn_box"]).abs().max() < 1e-4


@pytest.mark.parametrize("ragged", [False, True])
def test_full_transformer_forward_vs_reference(pkg, ragged):
    """Whole ``SalienceTransformer.forward`` (filter + encoder + two-stage selection + decoder), reference call signature and
    5-tuple of outputs.  Encoder memories differ by round-off, so near-tied proposals may swap: the proposal SETS must agree
    except for a few entries, and every query whose proposal agrees in position must agree in its outputs."""
    g, shapes = _golden(ragged)
    ours = _ours(pkg, shapes)
    feats, masks, pos = _inputs(ragged)
    want = [g[f"full{i}"] for i in range(4)] + [[g[f"full_score{i}"] for i in range(len([k for k in g if k.startswith("full_score")]))]]
    with torch.no_grad():
        pkg.gemm.MODE = "fp32"
        got = ours(feats, masks, pos, None, None, None)
    got = [t.cpu() for t in got[:4]] + [[t.cpu() for t in got[4]]]
    assert len(got) == 5 and got[0].shape == want[0].shape and got[1].shape == want[1].shape
    assert len(got[4]) == len(want[4])
    for a, w in zip(got[4], want[4]):  # salience score maps
        assert a.shape == w.shape and (a - w).abs().max() < 1e-4
    same = ((got[3] - want[3]).abs().amax(-1) < 1e-4)            # proposals equal position by position
    assert same.float().mean() > 0.9
    assert (got[2] - want[2]).abs().amax(-1)[same].max() < 1e-3   # their class logits
    if bool(same.all()):  # identical proposal lists: the decoder outputs must agree everywhere
        assert (got[0] - want[0]).abs().max() < 2e-3 and (got[1] - want[1]).abs().max() < 2e-4


def test_neck_handoff_vs_reference(pkg):
    """SURVEY.md 8(f)-3: the encoder memory is handed to a convolutional neck in per-level NCHW maps and comes back as tokens
    (salience_transformer.py:185-192).  Layout kernels: exact round trip; then a neck (oracle.ConvNeck, the reference's
    dict-of-levels interface) plugged into OUR transformer against the reference transformer with the same neck and weights:
    the memory that leaves the neck (captured at the decoder's `value` input) within 2e-3."""
    shapes = [(60, 80), (30, 40), (15, 20), (8, 10)]
    gen = torch.Generator().manual_seed(1)
    tok = torch.randn(2, sum(h * w for h, w in shapes), 96, generator=gen).to(DEV)
    maps = pkg.cabi.tokens_to_maps(tok, shapes)
    want = [t.transpose(1, 2).reshape(2, 96, h, w) for t, (h, w) in zip(tok.split([h * w for h, w in shapes], 1), shapes)]
    assert all(torch.equal(a, b) for a, b in zip(maps, want))
    assert torch.equal(pkg.cabi.maps_to_tokens(maps), tok)

    g, sd_shapes = _golden(False)
    ours = _ours(pkg, sd_shapes)
    ours.neck = orc.ConvNeck(GEO["embed_dim"], 4, seed=3).to(DEV).eval()
    feats, masks, pos = _inputs(False)
    cap = {}

    class _Stop(Exception):
        pass

    def grab(**kw):
        cap["value"] = kw["value"]
        raise _Stop()

    ours.decoder.forward = grab
    try:
        with torch.no_grad():
            pkg.gemm.MODE = "fp32"
            ours(feats, masks, pos, None, None, None)
    except _Stop:
        pass
    finally:
        del ours.decoder.forward
    idx = g["neck_rows_index"].to(DEV)
    a = torch.gather(cap["value"], 1, idx[..., None].expand(-1, -1, cap["value"].shape[2])).cpu()
    assert (a - g["neck_rows"]).abs().max() < 2e-3 * max(1.0, float(g["neck_value_absmax"]))
