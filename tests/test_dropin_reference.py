"""Drop-in tests against the UNMODIFIED reference modules on the GPU (row (b) of SURVEY.md section 8).

What the reference computes is stored in tests/golden/dropin_*.npz (oracle/make_golden.py runs the original project on the same
deterministic weights -- oracle.deterministic_state_dict -- and seeded inputs).  Three levels of "drops in unchanged":

1. operator: the MultiScaleDeformableAttention module (models/bricks/ms_deform_attn.py:286-377) on this package's
   forward / backward operator pair, against the reference module's forward and gradients;
2. module: this package's ``SalienceTransformerEncoder`` built from its layer class, as a reference config does
   (configs/salience_detr/salience_detr_resnet50_800_1333.py:44-62), fed the kwargs the reference's own filter
   (:106-168) hands to the encoder, against the reference encoder's memory;
3. transformer: this package's ``SalienceTransformer.forward_encoder`` with the reference's parameter names and weights,
   against the reference's filter outputs and memory.
"""
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
GEO = mg.DROPIN


@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


@pytest.fixture(autouse=True)
def _fp32_matmul(pkg):
    prev, mode = torch.backends.cuda.matmul.allow_tf32, pkg.gemm.MODE
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev
    pkg.gemm.MODE = mode


def _golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    g = {k: torch.from_numpy(z[k]) for k in z.files if k != "shapes_json"}
    return g, json.loads(str(z["shapes_json"]))


def _inputs(ragged):
    feats, masks, pos = orc.synthetic_inputs(mg.image_sizes(ragged), (480, 640), GEO["embed_dim"], seed=mg.DROPIN_INPUT_SEED)
    return [f.to(DEV) for f in feats], [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]


def _rows(mem, g):
    idx = g["memory_rows_index"].to(DEV)
    return torch.gather(mem, 1, idx[..., None].expand(-1, -1, mem.shape[2])).cpu()


def _transformer(pkg, shapes):
    """this package's encoder built from its layer class (what a reference config does) inside its SalienceTransformer, with the
    reference's parameter names and the fixture's weights"""
    layer = pkg.SalienceTransformerEncoderLayer(GEO["embed_dim"], GEO["d_ffn"], 0.0, GEO["n_heads"], torch.nn.ReLU(inplace=True),
                                                GEO["n_levels"], GEO["n_points"], topk_sa=GEO["topk_sa"])
    enc = pkg.SalienceTransformerEncoder(layer, GEO["num_layers"], max_num_embedding=GEO["max_num_embedding"])
    ours = pkg.SalienceTransformer(enc, None, None, GEO["num_classes"], GEO["n_levels"], GEO["num_proposals"],
                                   GEO["level_filter_ratio"], GEO["layer_filter_ratio"]).to(DEV).eval()
    res = ours.load_state_dict(orc.deterministic_state_dict(shapes, mg.DROPIN_SEED), strict=False)
    assert not res.unexpected_keys and all(k.endswith("_filter_ratio") for k in res.missing_keys)  # (constructor arguments)
    return ours


def _injected(pkg, ours, feats, masks, pos, plan, g, n_query):
    """this package's encoder on the reference filter's selection (the kwargs salience_transformer.py:161-183 passes)"""
    fg, inds = g["foreground_score"].to(DEV), g["selected_inds"].to(DEV)
    feat = pkg.flatten_levels(feats)
    lpos = pkg.flatten_levels([p + e.view(1, -1, 1, 1) for p, e in zip(pos, ours.level_embeds)])
    return ours.encoder(query=feat, query_pos=lpos, query_key_padding_mask=plan.mask_flat, spatial_shapes=plan.spatial_shapes,
                        level_start_index=plan.level_start_index, valid_ratios=plan.valid_ratios, foreground_score=fg,
                        focus_token_nums=plan.focus_token_nums, foreground_inds=[inds[:, :n] for n in n_query],
                        multi_level_masks=masks)


def test_operator_C_dropin_forward_backward(pkg):
    """The MSDA module on this package's forward / backward operator pair (the `_C` calls of ms_deform_attn.py:361-370) against the
    reference module's pure-PyTorch forward and gradients (query, value, sampling-offset and value-projection weights)."""
    g, shapes = _golden("dropin_msda_op")
    mod = pkg.MultiScaleDeformableAttention(256, 4, 8, 4).to(DEV)
    mod.load_state_dict(orc.deterministic_state_dict(shapes, mg.OP_SEED))
    query, refp, value, st, lsi, mask, gout = [t.to(DEV) for t in orc.dropin_msda_op_inputs()]
    query.requires_grad_(True), value.requires_grad_(True)
    n0 = pkg.cabi.launch_count()
    out = mod(query, refp, value, st, lsi, mask)
    grads = torch.autograd.grad(out, [query, value, mod.sampling_offsets.weight, mod.value_proj.weight], gout)
    assert pkg.cabi.launch_count() >= n0 + 2  # our forward and backward kernels really ran
    for i, (key, t) in enumerate(zip(("out", "g_query", "g_value", "g_offsets_w", "g_value_proj_w"), [out] + list(grads))):
        got = t.detach().reshape(-1)[g[key + "_idx"].to(DEV)].cpu()
        tol = 1e-4 if i == 0 else 1e-3 * max(1.0, float(g[key + "_absmax"]))
        assert (got - g[key]).abs().max() < tol, key


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("mode", ["fp32", "auto"])
def test_reference_transformer_with_our_encoder(pkg, ragged, mode):
    """This package's encoder, built from its layer class the way a reference config builds it, on the selection the reference's
    own filter made (identical tokens on both sides): memory within 1e-3 of the reference encoder's."""
    g, shapes = _golden("dropin_encoder_" + ("ragged" if ragged else "even"))
    feats, masks, pos = _inputs(ragged)
    ours = _transformer(pkg, shapes)
    assert ours.encoder.enhance_mcsp is ours.encoder_class_head  # injected by the constructor, as the reference does (:79)
    pkg.gemm.MODE = mode
    with torch.no_grad():
        plan = ours.make_plan(masks)
        n0 = pkg.cabi.launch_count()
        got = _injected(pkg, ours, feats, masks, pos, plan, g, g["layer_num_query"].tolist())
    assert pkg.cabi.launch_count() > n0 + 10
    err = (_rows(got, g) - g["memory_rows"]).abs().max().item()
    assert err < 1e-3, (mode, ragged, err)


@pytest.mark.parametrize("ragged", [False, True])
def test_our_transformer_with_reference_state_dict(pkg, ragged):
    """This package's SalienceTransformer (fused filter + encoder) loaded with the reference's parameters: the filter's budgets,
    scores and selection, and the memory, against the reference's."""
    g, shapes = _golden("dropin_encoder_" + ("ragged" if ragged else "even"))
    feats, masks, pos = _inputs(ragged)
    ours = _transformer(pkg, shapes)
    ref_inds, ref_fg = g["selected_inds"].to(DEV), g["foreground_score"].to(DEV)
    for mode, tol_score, swaps in (("fp32", 3e-5, 8), ("auto", 3e-4, 40)):
        pkg.gemm.MODE = mode
        with torch.no_grad():
            mem, aux = ours.forward_encoder(feats, masks, pos)
            plan = aux["plan"]
            assert plan.layer_num_query == g["layer_num_query"].tolist()
            assert torch.equal(plan.focus_token_nums.long().cpu(), g["focus_token_nums"].long())
            assert (aux["foreground_score"] - ref_fg).abs().max() < tol_score
            for i in range(2):
                n = int(plan.focus_host[i])
                a, w = set(aux["selected_inds"][i, :n].tolist()), set(ref_inds[i, :n].tolist())
                assert len(a & w) >= n - swaps, (mode, n - len(a & w))
            inj = _injected(pkg, ours, feats, masks, pos, plan, g, plan.layer_num_query)
        assert (_rows(inj, g) - g["memory_rows"]).abs().max() < 1e-3, mode
        if torch.equal(aux["selected_inds"], ref_inds):
            assert (_rows(mem, g) - g["memory_rows"]).abs().max() < 1e-3, mode
