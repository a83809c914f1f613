"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/*.npz by running the UNMODIFIED reference.

Run with a checkout of the original project:  SDETR_REFERENCE_ROOT=<its root> python oracle/make_golden.py
The reference ships no tests / golden vectors (SURVEY.md section 4); these fixtures are outputs of the
reference's own Python modules (imported via oracle/ref_import.py) on small seeded inputs, and are what
pins the oracle (tests/test_oracle_golden.py) and, through it, the CUDA kernels.

Fixtures
  msda_core_{a,b}.npz   multi_scale_deformable_attn_pytorch (ms_deform_attn.py:159-212) forward and its
                        autograd gradients (the contract of _C.ms_deform_attn_forward/backward).
  msda_module.npz       MultiScaleDeformableAttention.forward (ms_deform_attn.py:286-377) incl. state_dict.
  encoder_tiny_{even,ragged}.npz
                        SalienceTransformer.forward lines 106-183 (filter + encoder) of a tiny model:
                        inputs, encoder-half state_dict, the kwargs the filter hands to the encoder, and
                        the encoder memory.  "even": both images full size (tie-free selection);
                        "ragged": second image smaller (padded tokens -> ties, see SURVEY.md 8(a) notes).
  nms_topk.npz          SalienceTransformer.nms_on_topk_index (salience_transformer.py:249-295) on seeded candidate lists.
  dropin_msda_op.npz    MultiScaleDeformableAttention forward + gradients (sampled entries), deterministic weights.
  dropin_encoder_{even,ragged}.npz
                        filter outputs + sampled encoder memory of SalienceTransformer at the drop-in test geometry.
  decoder_half_{even,ragged}.npz
                        decoder outputs on seeded memory (with and without denoising queries), the whole forward's outputs,
                        and sampled memory behind a test neck.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle import oracle as orc  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def np_(t):
    return t.detach().cpu().numpy()


def make_msda_core(name, b, shapes, m, d, nq, p, seed):
    ref = ref_import.load()
    g = torch.Generator().manual_seed(seed)
    shapes_t = torch.tensor(shapes, dtype=torch.int64)
    nv = int(shapes_t.prod(1).sum())
    lsi = torch.cat([shapes_t.new_zeros(1), shapes_t.prod(1).cumsum(0)[:-1]])
    L = len(shapes)
    value = torch.randn(b, nv, m, d, generator=g, requires_grad=True)
    loc = (torch.rand(b, nq, m, L, p, 2, generator=g) * 1.2 - 0.1).requires_grad_(True)
    attn = torch.randn(b, nq, m, L * p, generator=g).softmax(-1).view(b, nq, m, L, p).requires_grad_(True)
    out = ref.msda.multi_scale_deformable_attn_pytorch(value, shapes_t, loc, attn)
    gout = torch.randn(out.shape, generator=g)
    gv, gl, ga = torch.autograd.grad(out, (value, loc, attn), gout)
    np.savez_compressed(os.path.join(OUT, name), value=np_(value), shapes=np_(shapes_t), lsi=np_(lsi),
                        loc=np_(loc), attn=np_(attn), out=np_(out), grad_out=np_(gout), grad_value=np_(gv),
                        grad_loc=np_(gl), grad_attn=np_(ga))


def make_msda_module(seed=3):
    ref = ref_import.load()
    torch.manual_seed(seed)
    mod = ref.msda.MultiScaleDeformableAttention(64, 4, 2, 4).eval()
    with torch.no_grad():  # non-trivial offsets / weights (init has zero weight matrices)
        mod.sampling_offsets.weight.normal_(0, 0.05)
        mod.attention_weights.weight.normal_(0, 0.5)
    shapes = [(9, 12), (5, 6), (3, 3), (2, 2)]
    shapes_t = torch.tensor(shapes)
    nv = int(shapes_t.prod(1).sum())
    lsi = torch.cat([shapes_t.new_zeros(1), shapes_t.prod(1).cumsum(0)[:-1]])
    b, nq = 2, 37
    query = torch.randn(b, nq, 64)
    refp = torch.rand(b, nq, 4, 2)
    value = torch.randn(b, nv, 64)
    mask = torch.rand(b, nv) < 0.15
    with torch.no_grad():
        out = mod(query, refp, value, shapes_t, lsi, mask)
    sd = {"sd." + k: np_(v) for k, v in mod.state_dict().items()}
    np.savez_compressed(os.path.join(OUT, "msda_module.npz"), query=np_(query), ref=np_(refp), value=np_(value),
                        shapes=np_(shapes_t), lsi=np_(lsi), mask=np_(mask), out=np_(out), **sd)


class _Stop(Exception):
    pass


TINY = dict(embed_dim=64, d_ffn=128, n_heads=2, n_levels=4, n_points=4, num_layers=3, num_classes=11,
            level_filter_ratio=(0.4, 0.8, 1.0, 1.0), layer_filter_ratio=(1.0, 0.6, 0.3), topk_sa=20,
            max_num_embedding=40, num_proposals=30)


def make_encoder_tiny(name, image_sizes, padded, seed):
    tr = ref_import.build_transformer(seed=seed, **TINY)
    with torch.no_grad():
        for layer in tr.encoder.layers:  # exercise learned offsets/weights, not only the init ring
            layer.self_attn.sampling_offsets.weight.normal_(0, 0.05)
            layer.self_attn.attention_weights.weight.normal_(0, 0.5)
    feats, masks, pos = orc.synthetic_inputs(image_sizes, padded, TINY["embed_dim"], seed=seed)
    captured = {}
    enc_fwd = tr.encoder.forward
    layer_out = []
    hooks = [l.register_forward_hook(lambda m, i, o: layer_out.append(o.detach().clone())) for l in tr.encoder.layers]

    def spy(**kw):
        captured.update(kw)
        captured["memory"] = enc_fwd(**kw)
        raise _Stop()

    tr.encoder.forward = spy
    try:
        with torch.no_grad():
            tr(feats, masks, pos, None, None, None)
    except _Stop:
        pass
    for h in hooks:
        h.remove()
    sd = {"sd." + k: np_(v) for k, v in tr.state_dict().items()
          if not (k.startswith("decoder") or k.startswith("tgt_embed") or k.startswith("encoder_bbox_head"))}
    arrs = {f"feat{i}": np_(f) for i, f in enumerate(feats)}
    arrs.update({f"mask{i}": np_(m) for i, m in enumerate(masks)})
    arrs.update({f"pos{i}": np_(p) for i, p in enumerate(pos)})
    arrs.update({f"layer_out{i}": np_(o) for i, o in enumerate(layer_out)})
    np.savez_compressed(
        os.path.join(OUT, name),
        memory=np_(captured["memory"]),
        foreground_score=np_(captured["foreground_score"]),
        focus_token_nums=np_(captured["focus_token_nums"]),
        selected_inds=np_(captured["foreground_inds"][0]),
        layer_num_query=np.array([x.shape[1] for x in captured["foreground_inds"]]),
        valid_ratios=np_(captured["valid_ratios"]),
        spatial_shapes=np_(captured["spatial_shapes"]),
        level_start_index=np_(captured["level_start_index"]),
        cfg_keys=np.array(sorted(TINY.keys())),
        **arrs, **sd)


def make_encoder_tiny_grads(name, image_sizes, padded, seed):
    """Gradients of the reference's own autograd through lines 106-183 for the tiny model of ``make_encoder_tiny`` (same
    seed -> same weights and inputs): d loss / d parameter for every parameter the loss reaches and d loss / d feats,
    loss = memory.square().mean().  Pins the training path (MSDA backward kernel inside torch autograd)."""
    tr = ref_import.build_transformer(seed=seed, **TINY).train()  # dropout = 0.0: train() only enables grad paths
    with torch.no_grad():
        for layer in tr.encoder.layers:
            layer.self_attn.sampling_offsets.weight.normal_(0, 0.05)
            layer.self_attn.attention_weights.weight.normal_(0, 0.5)
    feats, masks, pos = orc.synthetic_inputs(image_sizes, padded, TINY["embed_dim"], seed=seed)
    feats = [f.requires_grad_(True) for f in feats]
    captured = {}
    enc_fwd = tr.encoder.forward

    def spy(**kw):
        captured["memory"] = enc_fwd(**kw)
        raise _Stop()

    tr.encoder.forward = spy
    try:
        tr(feats, masks, pos, None, None, None)
    except _Stop:
        pass
    loss = captured["memory"].square().mean()
    loss.backward()
    out = {"loss": np_(loss)}
    for n, p in tr.named_parameters():
        if p.grad is not None:
            out["grad." + n] = np_(p.grad)
    for i, f in enumerate(feats):
        out[f"grad_feat{i}"] = np_(f.grad)
    np.savez_compressed(os.path.join(OUT, name), **out)


C256 = dict(embed_dim=256, d_ffn=256, n_heads=8, n_levels=4, n_points=4, num_layers=2, num_classes=11,
            level_filter_ratio=(0.4, 0.8, 1.0, 1.0), layer_filter_ratio=(1.0, 0.5), topk_sa=64,
            max_num_embedding=80, num_proposals=30)
C256_IMAGES, C256_PADDED, C256_SEED, C256_ROWS = [(384, 512), (384, 512)], (384, 512), 11, 256


def encoder_half_keys(state_dict):
    return {k: tuple(v.shape) for k, v in state_dict.items()
            if not (k.startswith("decoder") or k.startswith("tgt_embed") or k.startswith("encoder_bbox_head")
                    or k.endswith("_filter_ratio"))}


def make_encoder_c256(name="encoder_c256.npz"):
    """Reference width (C = 256, 8 heads of 32) at 4080 tokens per image: exercises the paths that are specialised for
    the real model (fused pre-attention, persistent tensor-core GEMM).  Weights come from
    oracle.deterministic_state_dict (regenerated by the tests), inputs from oracle.synthetic_inputs; the fixture holds
    the reference's outputs: selection, scores, and the encoder memory at C256_ROWS sampled tokens per image plus
    per-token channel means of all tokens."""
    import json
    tr = ref_import.build_transformer(seed=0, **C256)
    shapes = encoder_half_keys(tr.state_dict())
    missing = tr.load_state_dict(orc.deterministic_state_dict(shapes, C256_SEED), strict=False)
    assert not [k for k in missing.unexpected_keys]
    feats, masks, pos = orc.synthetic_inputs(C256_IMAGES, C256_PADDED, C256["embed_dim"], seed=C256_SEED)
    captured = {}
    enc_fwd = tr.encoder.forward

    def spy(**kw):
        captured.update(kw)
        captured["memory"] = enc_fwd(**kw)
        raise _Stop()

    tr.encoder.forward = spy
    try:
        with torch.no_grad():
            tr(feats, masks, pos, None, None, None)
    except _Stop:
        pass
    mem = captured["memory"]
    nv = mem.shape[1]
    rows = torch.stack([torch.randperm(nv, generator=torch.Generator().manual_seed(100 + i))[:C256_ROWS] for i in range(mem.shape[0])])
    np.savez_compressed(
        os.path.join(OUT, name),
        shapes_json=np.array(json.dumps({k: list(v) for k, v in shapes.items()})),
        memory_rows_index=np_(rows),
        memory_rows=np_(torch.gather(mem, 1, rows[..., None].expand(-1, -1, mem.shape[2]))),
        memory_row_mean=np_(mem.mean(-1)), memory_row_absmax=np_(mem.abs().amax(-1)),
        foreground_score=np_(captured["foreground_score"]),
        focus_token_nums=np_(captured["focus_token_nums"]),
        selected_inds=np_(captured["foreground_inds"][0]),
        layer_num_query=np.array([x.shape[1] for x in captured["foreground_inds"]]))


def make_salience_criterion(name="salience_criterion.npz"):
    """SalienceCriterion (models/detectors/salience_detr.py:13-116) + sigmoid_focal_loss (models/bricks/losses.py:4-12).
    The detector module cannot be imported here (pycocotools / accelerate are missing), so the two definitions are compiled
    from the reference's own source files, unmodified, without the modules' import lines; loss, its gradient w.r.t. the
    score maps, and the target maps on seeded boxes."""
    import ast
    from typing import Tuple  # noqa: F401
    from torch import nn
    from torch.nn import functional as F
    from torchvision.ops import boxes as box_ops
    ns = {"torch": torch, "nn": nn, "F": F, "box_ops": box_ops, "Tuple": Tuple}
    for path, kind, ident in ((os.path.join(ref_import.REFERENCE_ROOT, "models/bricks/losses.py"), ast.FunctionDef, "sigmoid_focal_loss"),
                              (os.path.join(ref_import.REFERENCE_ROOT, "models/detectors/salience_detr.py"), ast.ClassDef, "SalienceCriterion")):
        node = [n for n in ast.parse(open(path).read()).body if isinstance(n, kind) and n.name == ident][0]
        exec(compile(ast.Module(body=[node], type_ignores=[]), path, "exec"), ns)
    crit = ns["SalienceCriterion"]()
    g = torch.Generator().manual_seed(0)
    shapes = [(50, 84), (25, 42), (13, 21), (7, 11)]
    fg = [torch.randn(2, 1, h, w, generator=g).requires_grad_(True) for h, w in shapes]

    def boxes(n):
        return torch.cat([torch.rand(n, 2, generator=g) * 0.6 + 0.2, torch.rand(n, 2, generator=g) * 0.5 + 0.02], -1)

    targets = [{"boxes": boxes(7)}, {"boxes": boxes(3)}]
    image_sizes = [(400, 672), (380, 600)]
    strides = [(400 / h, 672 / w) for h, w in shapes]
    loss = crit(fg, targets, strides, image_sizes)["loss_salience"]
    loss.backward()
    mt = []
    for lvl, (shape, st) in enumerate(zip(shapes, strides)):
        cx, cy = crit.get_pixel_coordinate(shape, st, "cpu")
        mt.append(torch.stack([crit.get_mask_single_level(cx, cy, box_ops._box_cxcywh_to_xyxy(t["boxes"]) *
                                                          torch.tensor([iw, ih, iw, ih]), lvl)
                               for t, (ih, iw) in zip(targets, image_sizes)]))
    np.savez_compressed(os.path.join(OUT, name), loss=np_(loss), boxes0=np_(targets[0]["boxes"]), boxes1=np_(targets[1]["boxes"]),
                        image_sizes=np.array(image_sizes), shapes=np.array(shapes), strides=np.array(strides, dtype=np.float64),
                        mask_targets=np_(torch.cat(mt, 1)), **{f"fg{i}": np_(f) for i, f in enumerate(fg)},
                        **{f"grad{i}": np_(f.grad) for i, f in enumerate(fg)})


NMS_CASES = (([(60, 80), (30, 40), (15, 20), (8, 10)], 1200), ([(100, 168), (50, 84), (25, 42), (13, 21)], 3600),
             ([(20, 20), (10, 10)], 450))


def make_nms_topk(name="nms_topk.npz", seed=0):
    """Candidates: topk of torch.rand(2, Nv) scores drawn from manual_seed(seed) in case order (distinct with probability 1,
    so the order is unambiguous); kept = the reference's surviving token indices per image."""
    tr = ref_import.build_transformer(embed_dim=64, d_ffn=64, n_heads=2, num_layers=1, topk_sa=10, num_proposals=900)
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i, (shapes, k) in enumerate(NMS_CASES):
        st = torch.tensor(shapes)
        lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
        scores = torch.rand(2, int(st.prod(1).sum()), generator=g)
        topk_scores, topk_index = torch.topk(scores, k, dim=1)
        with torch.no_grad():
            out[f"kept{i}"] = np_(tr.nms_on_topk_index(topk_scores, topk_index, st, lsi, iou_threshold=0.3))
    np.savez_compressed(os.path.join(OUT, name), **out)


# ---- drop-in / decoder-half fixtures: what tests/test_dropin_reference.py and tests/test_decoder_half.py compare against ----
DROPIN = dict(embed_dim=256, d_ffn=512, n_heads=8, n_levels=4, n_points=4, num_layers=3, num_classes=17,
              level_filter_ratio=(0.4, 0.8, 1.0, 1.0), layer_filter_ratio=(1.0, 0.7, 0.4), topk_sa=100,
              max_num_embedding=100, num_proposals=50)
DROPIN_SEED, DROPIN_INPUT_SEED, DROPIN_ROWS = 21, 9, 128
HALF = dict(embed_dim=256, d_ffn=512, n_heads=8, num_layers=2, dec_layers=3, num_classes=17, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
            layer_filter_ratio=(1.0, 0.5), topk_sa=100, max_num_embedding=100, num_proposals=300)
HALF_SEED, HALF_INPUT_SEED, HALF_VALUE_SEED, HALF_ROWS = 22, 13, 31, 128
OP_SEED = 23


def image_sizes(ragged):
    return [(480, 640), (400, 500)] if ragged else [(480, 640), (480, 640)]


def sample_rows(mem, n, seed):
    """(b, Nv, C) -> (index (b, n), rows (b, n, C)): a fixed seeded choice of token rows per image"""
    rows = torch.stack([torch.randperm(mem.shape[1], generator=torch.Generator().manual_seed(seed + i))[:n] for i in range(mem.shape[0])])
    return rows, torch.gather(mem, 1, rows[..., None].expand(-1, -1, mem.shape[2]))


def sample_flat(t, n, seed):
    """a fixed seeded sample of n entries of t (flat indices, values) and max|t|"""
    idx = torch.randperm(t.numel(), generator=torch.Generator().manual_seed(seed))[:n]
    return np_(idx), np_(t.reshape(-1)[idx]), np.float32(t.abs().max().item())


def make_dropin_msda_op(name="dropin_msda_op.npz"):
    """MultiScaleDeformableAttention forward + gradients of the reference module (its pure-PyTorch core), deterministic weights."""
    import json
    ref = ref_import.load()
    mod = ref.msda.MultiScaleDeformableAttention(256, 4, 8, 4)
    shapes = {k: tuple(v.shape) for k, v in mod.state_dict().items()}
    mod.load_state_dict(orc.deterministic_state_dict(shapes, OP_SEED))
    query, refp, value, st, lsi, mask, gout = orc.dropin_msda_op_inputs()
    query.requires_grad_(True), value.requires_grad_(True)
    out = mod(query, refp, value, st, lsi, mask)
    grads = torch.autograd.grad(out, [query, value, mod.sampling_offsets.weight, mod.value_proj.weight], gout)
    res = {"shapes_json": np.array(json.dumps({k: list(v) for k, v in shapes.items()}))}
    for i, (key, t) in enumerate(zip(("out", "g_query", "g_value", "g_offsets_w", "g_value_proj_w"), [out] + list(grads))):
        res[key + "_idx"], res[key], res[key + "_absmax"] = sample_flat(t.detach(), 4096, 500 + i)
    np.savez_compressed(os.path.join(OUT, name), **res)


def make_dropin_encoder(ragged):
    """Reference SalienceTransformer (filter + encoder) at the drop-in geometry: the kwargs its filter hands to the encoder and the
    encoder memory at DROPIN_ROWS sampled tokens per image."""
    import json
    tr = ref_import.build_transformer(seed=0, **DROPIN)
    shapes = encoder_half_keys(tr.state_dict())
    tr.load_state_dict(orc.deterministic_state_dict(shapes, DROPIN_SEED), strict=False)
    feats, masks, pos = orc.synthetic_inputs(image_sizes(ragged), (480, 640), 256, seed=DROPIN_INPUT_SEED)
    mem, kw = ref_import.run_encoder_half(tr, feats, masks, pos)
    rows, vals = sample_rows(mem, DROPIN_ROWS, 200)
    np.savez_compressed(
        os.path.join(OUT, "dropin_encoder_%s.npz" % ("ragged" if ragged else "even")),
        shapes_json=np.array(json.dumps({k: list(v) for k, v in shapes.items()})),
        memory_rows_index=np_(rows), memory_rows=np_(vals), foreground_score=np_(kw["foreground_score"]),
        focus_token_nums=np_(kw["focus_token_nums"]), selected_inds=np_(kw["foreground_inds"][0]),
        layer_num_query=np.array([x.shape[1] for x in kw["foreground_inds"]]))


def half_reference():
    """Reference SalienceTransformer with a HALF["dec_layers"]-layer decoder and deterministic weights (all parameters)."""
    ref = ref_import.load()
    st, relu, H = ref.st, torch.nn.ReLU(inplace=True), HALF
    enc = st.SalienceTransformerEncoder(st.SalienceTransformerEncoderLayer(H["embed_dim"], H["d_ffn"], 0.0, H["n_heads"], relu, 4, 4,
                                                                           topk_sa=H["topk_sa"]), H["num_layers"],
                                        max_num_embedding=H["max_num_embedding"])
    dec = st.SalienceTransformerDecoder(st.SalienceTransformerDecoderLayer(H["embed_dim"], H["d_ffn"], H["n_heads"], 0.0, relu, 4, 4),
                                        H["dec_layers"], H["num_classes"])
    tr = st.SalienceTransformer(enc, None, dec, H["num_classes"], 4, H["num_proposals"], H["level_filter_ratio"], H["layer_filter_ratio"])
    shapes = {k: tuple(v.shape) for k, v in tr.state_dict().items() if not k.endswith("_filter_ratio")}
    tr.load_state_dict(orc.deterministic_state_dict(shapes, HALF_SEED), strict=False)
    return tr.eval(), shapes


def make_decoder_half(ragged):
    """Reference decoder on seeded memory (with the filter's masks / ratios / proposals of the real forward), with and without
    denoising queries; the whole forward's five outputs; the memory leaving an oracle.ConvNeck at the decoder's `value` input."""
    import json
    tr, shapes = half_reference()
    feats, masks, pos = orc.synthetic_inputs(image_sizes(ragged), (480, 640), 256, seed=HALF_INPUT_SEED)
    cap = {}
    dec_fwd = tr.decoder.forward

    def spy(**kw):
        cap.update(kw)
        return dec_fwd(**kw)

    tr.decoder.forward = spy
    with torch.no_grad():
        full = tr(feats, masks, pos, None, None, None)
    del tr.decoder.forward
    kw = {k: v for k, v in cap.items()}
    kw["value"] = orc.seeded_memory(kw["value"].shape, HALF_VALUE_SEED)
    dn_q, dn_b, attn_mask = orc.denoising_queries(kw["query"].shape[0], kw["query"].shape[1], HALF["embed_dim"])
    kw2 = dict(kw, query=torch.cat([dn_q, kw["query"]], 1), reference_points=torch.cat([dn_b, kw["reference_points"]], 1),
               attn_mask=attn_mask)
    with torch.no_grad():
        cls, box = tr.decoder(**kw)
        cls2, box2 = tr.decoder(**kw2)
    neck_cap = {}
    tr.neck = orc.ConvNeck(HALF["embed_dim"], 4, seed=3)

    def grab(**k):
        neck_cap["value"] = k["value"]
        raise _Stop()

    tr.decoder.forward = grab
    try:
        with torch.no_grad():
            tr(feats, masks, pos, None, None, None)
    except _Stop:
        pass
    del tr.decoder.forward
    rows, vals = sample_rows(neck_cap["value"], HALF_ROWS, 300)
    res = dict(shapes_json=np.array(json.dumps({k: list(v) for k, v in shapes.items()})),
               reference_points=np_(kw["reference_points"]), key_padding_mask=np_(kw["key_padding_mask"]),
               valid_ratios=np_(kw["valid_ratios"]), spatial_shapes=np_(kw["spatial_shapes"]),
               level_start_index=np_(kw["level_start_index"]), dec_cls=np_(cls), dec_box=np_(box), dn_cls=np_(cls2), dn_box=np_(box2),
               neck_rows_index=np_(rows), neck_rows=np_(vals), neck_value_absmax=np.float32(neck_cap["value"].abs().max().item()))
    for i, t in enumerate(full[:4]):
        res[f"full{i}"] = np_(t)
    for i, t in enumerate(full[4]):
        res[f"full_score{i}"] = np_(t)
    np.savez_compressed(os.path.join(OUT, "decoder_half_%s.npz" % ("ragged" if ragged else "even")), **res)


def main():
    os.makedirs(OUT, exist_ok=True)
    make_msda_core("msda_core_a.npz", b=2, shapes=[(10, 12), (5, 6), (3, 3), (2, 2)], m=4, d=32, nq=40, p=4, seed=1)
    make_msda_core("msda_core_b.npz", b=1, shapes=[(7, 5), (4, 3)], m=2, d=16, nq=23, p=2, seed=2)
    make_msda_module()
    make_encoder_tiny("encoder_tiny_even.npz", [(96, 128), (96, 128)], (96, 128), seed=5)
    make_encoder_tiny("encoder_tiny_ragged.npz", [(96, 128), (72, 90)], (96, 128), seed=6)
    make_encoder_c256()
    make_encoder_tiny_grads("encoder_tiny_even_grads.npz", [(96, 128), (96, 128)], (96, 128), seed=5)
    make_salience_criterion()
    make_nms_topk()
    make_dropin_msda_op()
    for ragged in (False, True):
        make_dropin_encoder(ragged)
        make_decoder_half(ragged)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")
    print("torch", torch.__version__)


if __name__ == "__main__":
    main()
