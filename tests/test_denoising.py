"""GenerateCDNQueries / compute_dn_loss on the GPU (salience-detr_b200/denoising.py, csrc/denoising.cu) against the fixture made
from the unmodified reference (tests/golden/cdn_queries.npz, tools/make_cdn_golden.py) and the plain-torch restatement in
oracle/denoising.py."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import denoising as odn
from oracle import set_criterion as osc

gpu = pytest.mark.gpu
NAMES = list(odn.CASES)


def _pkg():
    import salience_detr_b200 as pkg
    return pkg


def fixture():
    return np.load(os.path.join(GOLDEN, "cdn_queries.npz"))


def case(z, name):
    seed = int(z["seed"]) + NAMES.index(name)
    labels, boxes, cfg = odn.case_inputs(name, seed)
    draws = tuple(torch.from_numpy(z[f"{name}.{k}"]) if f"{name}.{k}" in z.files else None
                  for k in ("label_rand", "label_randint", "box_randint", "box_rand"))
    return seed, labels, boxes, cfg, draws


def bits(t):
    t = t.detach().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same_bits(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def oracle_run(z, name, device="cpu"):
    seed, labels, boxes, cfg, draws = case(z, name)
    nq, K, C, dn, p, s = cfg
    w = torch.from_numpy(z[f"{name}.weight"]).to(device).requires_grad_(True)
    out = odn.cdn_queries(w, [x.to(device) for x in labels], [x.to(device) for x in boxes], nq, K, dn, p, s,
                          [d.to(device) if d is not None else None for d in draws])
    up = torch.randn(out[0].shape, generator=torch.Generator().manual_seed(seed + 1)).to(device)
    if out[0].requires_grad:
        (out[0] * up).sum().backward()
    return out, w.grad if w.grad is not None else torch.zeros_like(w)


# ---- CPU --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_fixture_bit_for_bit(name):
    z = fixture()
    (lq, bq, mask, groups, max_gt, _, _), gw = oracle_run(z, name)
    assert same_bits(lq, torch.from_numpy(z[f"{name}.label_queries"]))
    assert same_bits(bq, torch.from_numpy(z[f"{name}.box_queries"]))
    assert same_bits(mask, torch.from_numpy(z[f"{name}.attn_mask"]))
    assert groups == int(z[f"{name}.groups"]) and max_gt == int(z[f"{name}.max_gt"])
    assert same_bits(gw, torch.from_numpy(z[f"{name}.weight_grad"]))


def test_fixture_reaches_every_clamp():
    """the edge case hits clamp(0, 1) of the noised corners and both eps clamps of inverse_sigmoid"""
    z = fixture()
    bq = torch.from_numpy(z["edges.box_queries"])
    lim = float(np.log(np.float32(1e-3) / np.float32(1 - np.float32(1e-3))))
    assert (bq <= lim + 1e-6).any() and (bq >= -lim - 1e-6).any()


def test_initial_weights_and_keys_match_reference():
    pkg = _pkg()
    z = fixture()
    torch.manual_seed(odn.INIT["seed"])
    m = pkg.GenerateCDNQueries(*odn.INIT["cfg"])
    sd = m.state_dict()
    want = {k[5:]: z[k] for k in z.files if k.startswith("init.")}
    assert sorted(sd) == sorted(want) == ["label_encoder.weight"]
    assert same_bits(sd["label_encoder.weight"], torch.from_numpy(want["label_encoder.weight"]))
    nq, K, C, dn, p, s = odn.INIT["cfg"]
    assert (m.num_queries, m.num_classes, m.label_embed_dim, m.denoising_nums, m.label_noise_prob, m.box_noise_scale,
            m.denoising_groups, m.with_indicator) == (nq, K, C, dn, p, s, 1, False)


@pytest.mark.parametrize("name", NAMES)
def test_mirror_draws_like_the_reference(name):
    """Same seed: the mirror's construction then its draws give the reference's weights and the reference's random tensors
    (same calls, order and shapes; on the CPU generator here)."""
    pkg = _pkg()
    z = fixture()
    seed, labels, boxes, cfg, draws = case(z, name)
    torch.manual_seed(seed)
    m = pkg.GenerateCDNQueries(*cfg)
    assert same_bits(m.label_encoder.weight, torch.from_numpy(z[f"{name}.weight"]))
    g = odn.groups_of([x.numel() for x in labels], cfg[3])
    got = m.draws(2 * g * sum(x.numel() for x in labels), "cpu")
    for a, b in zip(got, draws):
        assert (a is None) == (b is None)
        if a is not None:
            assert same_bits(a, b)


def test_cpu_inputs_raise():
    pkg = _pkg()
    m = pkg.GenerateCDNQueries(20, 11, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        m([torch.tensor([1, 2])], [torch.rand(2, 4)])


def test_cabi_rejects_bad_arguments():
    """Every call below is refused on the host before any CUDA call (the pointers are never dereferenced)."""
    pkg = _pkg()
    import __graft_entry__ as entry
    entry.build()
    lib, Im = pkg.cabi.lib(), pkg.cabi.CDNImage
    fake = 256

    def q(ims, count=None, K=11, C=16, rows=11, cols=16, weight=fake, groups=14, max_gt=7, draws=(fake,) * 4, label_q=fake,
          mask=fake, status=fake):
        tab = (Im * max(len(ims), 1))(*ims)
        return lib.sdetr_cdn_queries(tab if ims else None, len(ims) if count is None else count, *draws, 0.25, 1.0, weight, K, C,
                                     rows, cols, 20, groups, max_gt, label_q, fake, fake, mask, status, None)

    ok = [Im(gt_labels=fake, gt_boxes=fake, num_gt=3), Im(gt_labels=fake, gt_boxes=fake, num_gt=7)]
    err = lambda: lib.sdetr_last_error()  # noqa: E731
    assert q([Im(gt_labels=None, gt_boxes=fake, num_gt=3)] + ok[1:]) == -1 and b"null pointer" in err()
    assert q([Im(gt_labels=fake, gt_boxes=None, num_gt=3)] + ok[1:]) == -1 and b"gt_boxes" in err()
    assert q([], count=2) == -1 and b"null pointer" in err()
    assert q([Im(gt_labels=fake, gt_boxes=fake, num_gt=-1)] + ok[1:]) == -1 and b"-1 gts" in err()
    assert q(ok * 65) == -1 and b"0..128" in err()
    assert q(ok, count=-1) == -1
    assert q(ok, rows=12) == -1 and b"label_encoder.weight is (12, 16)" in err()
    assert q(ok, cols=15) == -1 and b"expected (num_classes 11, embed_dim 16)" in err()
    assert q(ok, weight=None) == -1 and b"null pointer" in err()
    assert q(ok, label_q=None) == -1 and b"null pointer" in err()
    assert q(ok, mask=None) == -1 and q(ok, status=None) == -1
    assert q(ok, max_gt=6) == -1 and b"largest gt count is 7" in err()
    assert q(ok, groups=0) == -1
    assert q(ok, draws=(fake, None, fake, fake)) == -1 and b"both label draws" in err()
    assert q(ok, draws=(None, None, fake, fake)) == -1 and b"draws are missing" in err()
    # backward and loss indices
    assert lib.sdetr_cdn_queries_backward(fake, fake, 10, 0, 16, fake, None) == -1
    assert lib.sdetr_cdn_queries_backward(fake, fake, -1, 11, 16, fake, None) == -1
    assert lib.sdetr_cdn_queries_backward(None, fake, 10, 11, 16, fake, None) == -1 and b"null pointer" in err()
    assert lib.sdetr_cdn_queries_backward(fake, fake, 10, 11, 16, None, None) == -1
    counts = pkg.cabi._host_i32([3, 7])
    assert lib.sdetr_cdn_loss_indices(None, 2, 14, 14, fake, None) == -1 and b"null pointer" in err()
    assert lib.sdetr_cdn_loss_indices(counts, 129, 14, 14, fake, None) == -1 and b"0..128" in err()
    assert lib.sdetr_cdn_loss_indices(pkg.cabi._host_i32([3, -7]), 2, 14, 14, fake, None) == -1 and b"-7 gts" in err()
    assert lib.sdetr_cdn_loss_indices(counts, 2, 14, 6, fake, None) == -1 and b"max_gt 6" in err()
    assert lib.sdetr_cdn_loss_indices(counts, 2, 14, 14, None, None) == -1 and b"null pointer" in err()
    assert lib.sdetr_cdn_loss_indices(counts, 2, 0, 14, fake, None) == -1


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def _module(z, name, cfg):
    pkg = _pkg()
    m = pkg.GenerateCDNQueries(*cfg).cuda()
    with torch.no_grad():
        m.label_encoder.weight.copy_(torch.from_numpy(z[f"{name}.weight"]))
    return m


@gpu
@pytest.mark.parametrize("name", NAMES)
def test_kernel_matches_fixture(name):
    pkg = _pkg()
    z = fixture()
    seed, labels, boxes, cfg, draws = case(z, name)
    nq, K, C, dn, p, s = cfg
    m = _module(z, name, cfg)
    counts = [x.numel() for x in labels]
    G, mx = odn.groups_of(counts, dn), max(counts)
    lq, bq, noised, mask, status = pkg.cabi.cdn_queries([x.cuda() for x in labels], [x.cuda() for x in boxes],
                                                        [d.cuda() if d is not None else None for d in draws],
                                                        m.label_encoder.weight.detach(), K, C, p * 0.5, s, nq, G, mx)
    assert same_bits(lq, torch.from_numpy(z[f"{name}.label_queries"]))
    assert same_bits(mask, torch.from_numpy(z[f"{name}.attn_mask"]))
    assert not status.any()
    # Boxes: the fixture's CPU arithmetic with torch's CUDA log in inverse_sigmoid (the reference's log on the GPU), bit for bit.
    # torch's CPU and CUDA log of the same float32 argument can differ in the last bit; that is the only allowed difference.
    want = odn.cdn_queries(torch.from_numpy(z[f"{name}.weight"]), labels, boxes, nq, K, dn, p, s, draws,
                           log=lambda x: torch.log(x.cuda()).cpu())[1]
    assert same_bits(bq, want)
    fix = torch.from_numpy(z[f"{name}.box_queries"])
    ulps = (bits(bq).long() - bits(fix).long()).abs()
    print(f"{name}: {int((ulps > 0).sum())} of {fix.numel()} box entries differ from the CPU fixture, by at most "
          f"{int(ulps.max()) if fix.numel() else 0} ulp (CPU vs CUDA log)")
    assert fix.numel() == 0 or int(ulps.max()) <= 1
    assert (G, 2 * mx) == (int(z[f"{name}.groups"]), int(z[f"{name}.max_gt"]))
    # the noised labels the backward uses: the gathered rows are the weight rows of these labels, -1 in padding slots
    w = m.label_encoder.weight.detach()
    nl = noised.long()
    assert torch.equal(lq[nl >= 0], w[nl[nl >= 0]]) and not lq[nl < 0].any()


@gpu
@pytest.mark.parametrize("name", ["counts_3_7", "m1_g100", "m120_g1", "empty_image", "all_empty", "no_noise"])
def test_forward_matches_oracle_on_cuda_from_the_same_seed(name):
    z = fixture()
    seed, labels, boxes, cfg, _ = case(z, name)
    nq, K, C, dn, p, s = cfg
    m = _module(z, name, cfg)
    labels, boxes = [x.cuda() for x in labels], [x.cuda() for x in boxes]
    torch.cuda.manual_seed(seed)
    got = m(labels, boxes)
    state_got = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(seed)
    want = odn.cdn_queries(m.label_encoder.weight.detach(), labels, boxes, nq, K, dn, p, s)
    state_want = torch.cuda.get_rng_state()
    for a, b in zip(got[:3], want[:3]):
        assert same_bits(a, b)
    assert got[3:] == want[3:5] and m.denoising_groups == want[3]
    assert torch.equal(state_got, state_want)  # the same random numbers were consumed
    assert not m.status.any()


def _grads(m, labels, boxes, seed, up):
    m.label_encoder.weight.grad = None
    torch.cuda.manual_seed(seed)
    lq = m(labels, boxes)[0]
    (lq * up).sum().backward()
    return m.label_encoder.weight.grad.clone()


@gpu
@pytest.mark.parametrize("name", ["counts_3_7", "m1_g100", "m120_g1", "edges"])
def test_weight_gradient(name):
    """within 1e-6 of torch autograd through the oracle (summation order only); bit-identical run to run, with and without
    torch.use_deterministic_algorithms(True)"""
    z = fixture()
    seed, labels, boxes, cfg, _ = case(z, name)
    nq, K, C, dn, p, s = cfg
    m = _module(z, name, cfg)
    labels, boxes = [x.cuda() for x in labels], [x.cuda() for x in boxes]
    torch.cuda.manual_seed(seed)
    shape = m(labels, boxes)[0].shape
    up = torch.randn(shape, generator=torch.Generator().manual_seed(seed + 1)).cuda()
    runs = [_grads(m, labels, boxes, seed, up) for _ in range(2)]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs.append(_grads(m, labels, boxes, seed, up))
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(same_bits(r, runs[0]) for r in runs)
    w = m.label_encoder.weight.detach().clone().requires_grad_(True)
    torch.cuda.manual_seed(seed)
    lq = odn.cdn_queries(w, labels, boxes, nq, K, dn, p, s)[0]
    (lq * up).sum().backward()
    err = ((runs[0] - w.grad).abs().max() / w.grad.abs().max()).item()
    print(f"{name}: weight grad rel err {err:.2e}")
    assert err <= 1e-6


@gpu
def test_no_sync_and_constant_launches():
    """forward + backward + the loss indices under set_sync_debug_mode("error"): one library launch each"""
    pkg = _pkg()
    z = fixture()
    counts = []
    for name in ("counts_3_7", "m1_g100"):
        seed, labels, boxes, cfg, _ = case(z, name)
        m = _module(z, name, cfg)
        labels, boxes = [x.cuda() for x in labels], [x.cuda() for x in boxes]
        m(labels, boxes)  # warm-up
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            n0 = pkg.cabi.launch_count()
            lq, bq, mask, G, m2 = m(labels, boxes)
            n1 = pkg.cabi.launch_count()
            lq.sum().backward()
            n2 = pkg.cabi.launch_count()
            pkg.cabi.cdn_loss_indices([x.numel() for x in labels], G, m2, "cuda")
            n3 = pkg.cabi.launch_count()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        counts.append((n1 - n0, n2 - n1, n3 - n2))
    assert counts == [(1, 1, 1)] * 2


@gpu
def test_graph_capture_replays_like_eager():
    z = fixture()
    seed, labels, boxes, cfg, _ = case(z, "counts_3_7")
    m = _module(z, "counts_3_7", cfg)
    labels, boxes = [x.cuda() for x in labels], [x.cuda() for x in boxes]
    with torch.no_grad():
        shape = m(labels, boxes)[0].shape
    up = torch.randn(shape, generator=torch.Generator().manual_seed(5)).cuda()

    def step():
        m.label_encoder.weight.grad = None
        lq, bq, mask, _, _ = m(labels, boxes)
        (lq * up).sum().backward()
        return [lq.detach(), bq, mask, m.label_encoder.weight.grad]  # nothing keeps the autograd graph alive

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for sd in (21, 22):
        torch.cuda.manual_seed(sd)
        graph.replay()
        got = [t.clone() for t in static]
        torch.cuda.manual_seed(sd)
        eager = step()
        assert all(same_bits(a, b) for a, b in zip(got, eager))


@gpu
def test_label_out_of_range_gives_nan_and_status():
    pkg = _pkg()
    m = pkg.GenerateCDNQueries(20, 11, 16, 100, 0.0, 1.0).cuda()  # no label noise: the bad label survives
    g = torch.Generator().manual_seed(2)
    labels = [torch.tensor([1, 11, 4]).cuda(), torch.tensor([0, 10]).cuda()]
    boxes = [osc.random_boxes(g, 3).cuda(), osc.random_boxes(g, 2).cuda()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        lq, bq, mask, G, m2 = m(labels, boxes)
        lq.sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m.status.tolist() == [1, 0]
    bad = torch.zeros(2, lq.shape[1], dtype=torch.bool)
    bad[0, torch.arange(2 * G) * 3 + 1] = True
    nan_rows = torch.isnan(lq).all(-1).cpu()
    assert torch.equal(nan_rows, bad) and torch.isfinite(lq.cpu()[~bad]).all()
    assert torch.isfinite(bq).all() and torch.isfinite(m.label_encoder.weight.grad).all()


@gpu
@pytest.mark.parametrize("dn_nums", [100, 20])
def test_compute_dn_loss_matches_per_output_calls_through_the_decoder(dn_nums):
    """The decoder's real outputs (HALF geometry, as tests/test_set_criterion.py) with this generator's denoising queries in
    front: compute_dn_loss gives the losses of one calculate_loss(indices=...) call per denoising output, built as the
    reference builds them (meshgrid indices, num_boxes * groups), bit for bit -- each output's sum is reduced on its own in a
    fixed order, so batching changes no summation order.  label_encoder.weight receives a gradient through the decoder."""
    pkg = _pkg()
    import test_set_criterion as tsc
    from oracle import make_golden as mg
    from oracle import oracle as orc
    ttg = tsc._training_gradients()
    tdh = ttg._decoder_half()
    g, shapes = tdh._golden(False)
    ours = tdh._ours(pkg, shapes).train()
    b = g["reference_points"].shape[0]
    nv = int(g["key_padding_mask"].shape[1])
    dev = ttg.DEV
    K, C = mg.HALF["num_classes"], mg.HALF["embed_dim"]
    torch.manual_seed(17)
    gen = pkg.GenerateCDNQueries(300, K, C, dn_nums, 0.5, 1.0).to(dev)
    rg = torch.Generator().manual_seed(13)
    gt_counts = (5, 3)[:b] + (4,) * max(b - 2, 0)
    targets = [{"boxes": osc.random_boxes(rg, n).to(dev), "labels": torch.randint(0, K, (n,), generator=rg).to(dev)}
               for n in gt_counts]
    torch.cuda.manual_seed(3)
    lq, bq, mask, G, m2 = gen([t["labels"] for t in targets], [t["boxes"] for t in targets])
    pad = lq.shape[1]
    kw = dict(query=torch.cat([lq, ours.tgt_embed.weight.detach().expand(b, -1, -1)], 1),
              value=orc.seeded_memory((b, nv, C), mg.HALF_VALUE_SEED).to(dev), key_padding_mask=g["key_padding_mask"].to(dev),
              reference_points=torch.cat([bq.sigmoid(), g["reference_points"].to(dev)], 1),
              spatial_shapes=g["spatial_shapes"].to(dev), level_start_index=g["level_start_index"].to(dev),
              valid_ratios=g["valid_ratios"].to(dev), attn_mask=mask)
    cls, box = ours.decoder(**kw)
    _, dn = tsc._split_like_dn_post_process(cls, box, pad)
    dn_metas = {"denoising_groups": G, "max_gt_num_per_image": m2, "denoising_output": dn}
    crit = tsc._criterion(K, False)
    got = pkg.compute_dn_loss(crit, dn_metas, targets)
    # DNDETRDetector.compute_dn_loss as the reference writes it, with this package's calculate_loss per output
    nb = torch.clamp(torch.as_tensor([float(sum(gt_counts))], device=dev), min=1).item()
    idx = []
    for t in targets:
        gi, ti = torch.meshgrid(torch.arange(G, device=dev), torch.arange(len(t["labels"]), device=dev), indexing="ij")
        idx.append(((gi * m2 + ti).flatten(), ti.flatten()))
    want = {}
    for j, o in enumerate([dn] + dn["aux_outputs"]):
        suf = "_dn" if j == 0 else f"_dn_{j - 1}"
        want.update({k + suf: v for k, v in crit.calculate_loss(o, targets, num_boxes=nb * G, indices=idx).items()})
    assert list(got) == list(want) and len(got) == 3 * mg.HALF["dec_layers"]
    for k in want:
        assert same_bits(got[k], want[k]), k
    # and the plain-torch chain (oracle, float32 on the GPU) within float32 round-off
    ref = odn.dn_loss(dn_metas, targets)
    for k in want:
        a, r = got[k].item(), ref[k].item()
        assert abs(a - r) <= 1e-5 * abs(r) + 1e-7, k
    sum(got.values()).backward()
    gw = gen.label_encoder.weight.grad
    assert gw is not None and torch.isfinite(gw).all() and gw.abs().sum() > 0
