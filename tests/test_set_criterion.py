"""HungarianMatcher / HybridSetCriterion on the GPU (salience-detr_b200/set_criterion.py, csrc/set_criterion.cu) against
scipy, the plain-torch restatement in oracle/set_criterion.py and the fixtures made from the reference
(tools/make_set_criterion_golden.py)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import set_criterion as osc

gpu = pytest.mark.gpu
CASES = {  # tools/make_set_criterion_golden.py CASES (inputs are regenerated from the stored seed)
    "small": dict(bs=2, Q=300, K=20, gt_counts=(7, 30), num_aux=1, enc_q=300, binary=True, tie=False, dn=0),
    "c2": dict(bs=2, Q=900, K=91, gt_counts=(100, 0), num_aux=5, enc_q=850, binary=False, tie=True, dn=100),
}


def fixture(name):
    z = np.load(os.path.join(GOLDEN, f"set_criterion_{name}.npz"))
    cfg = CASES[name]
    outputs, targets, dn = osc.synthetic_case(int(z["seed"]), cfg["bs"], cfg["Q"], cfg["K"], cfg["gt_counts"], cfg["num_aux"],
                                              cfg["enc_q"], cfg["dn"], cfg["tie"])
    return z, cfg, outputs, targets, dn


def rel(a, b):
    a = a.detach() if torch.is_tensor(a) else a
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-12)


def grad_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want).max() / max(np.abs(want).max(), 1e-30)


def check_grads(z, suf, out_grads, tol):
    gl, gb = out_grads
    assert grad_err(gb, z[f"gb{suf}"]) < tol, suf
    if f"gl_pos{suf}" in z.files:
        assert grad_err(gl.reshape(-1)[z[f"gl_pos{suf}"]], z[f"gl{suf}"]) < tol, suf
    else:
        assert grad_err(gl, z[f"gl{suf}"]) < tol, suf


# ---- CPU: the oracle restatement reproduces the reference fixtures --------------------------------------------------------
@pytest.mark.parametrize("name", ["small", "c2"])
def test_oracle_reproduces_fixture(name):
    pytest.importorskip("scipy")
    z, cfg, outputs, targets, dn = fixture(name)
    _, idx = osc.criterion(outputs, targets, cfg["binary"])  # fp32 costs, as the reference matches in training
    for suf, ind in idx.items():
        for i, (s, t) in enumerate(ind):
            assert np.array_equal(s.numpy(), z[f"src{suf}_{i}"]) and np.array_equal(t.numpy(), z[f"tgt{suf}_{i}"]), (suf, i)
    out64 = osc.to_dtype(outputs, torch.float64, requires_grad=True)
    tg64 = [dict(t, boxes=t["boxes"].double()) for t in targets]
    losses, idx64 = osc.criterion(out64, tg64, cfg["binary"])
    assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for k in idx for a, b in zip(idx[k], idx64[k]))
    for k, v in losses.items():
        assert rel(v, z["loss." + k]) < 1e-6, k
    sum(losses.values()).backward()
    for suf, o in osc.flat_outputs(out64):
        check_grads(z, suf, (o["pred_logits"].grad.numpy(), o["pred_boxes"].grad.numpy()), 1e-6)
    if dn is not None:
        dn64 = osc.to_dtype(dn, torch.float64, requires_grad=True)
        ind = osc.dn_indices(targets, int(z["dn.groups"]), int(z["dn.max_gt"]))
        dl = osc.calculate_loss(dn64["pred_logits"], dn64["pred_boxes"], tg64, osc.num_boxes_of(targets) * int(z["dn.groups"]),
                                ind)
        for k, v in dl.items():
            assert rel(v, z["dn." + k]) < 1e-6, k
        sum(dl.values()).backward()
        assert grad_err(dn64["pred_logits"].grad.numpy(), z["dn.gl"]) < 1e-6
        assert grad_err(dn64["pred_boxes"].grad.numpy(), z["dn.gb"]) < 1e-6


# ---- CPU: host-side rules ------------------------------------------------------------------------------------------------------
def test_host_packing_and_num_boxes():
    import salience_detr_b200.set_criterion as sc

    assert sc.pair_offsets([3, 0, 100, 7]) == [0, 3, 3, 103]
    assert sc.pair_offsets([]) == []
    t = lambda n: {"labels": torch.zeros(n, dtype=torch.int64), "boxes": torch.zeros(n, 4)}  # noqa: E731
    # SetCriterion.forward: clamp(sum(len(labels)) / world_size, min=1) -- all-empty targets give 1
    assert sc.num_boxes_of([t(0), t(0)]) == 1.0 == osc.num_boxes_of([t(0), t(0)])
    assert sc.num_boxes_of([t(7), t(0), t(30)]) == 37.0 == osc.num_boxes_of([t(7), t(0), t(30)])
    with pytest.raises(NotImplementedError, match="mixed_match"):
        sc.HungarianMatcher(2, 5, 2, mixed_match=True)


def test_cabi_rejects_bad_problems():
    """Every call below is refused on the host before any CUDA call (the pointers are never dereferenced)."""
    import salience_detr_b200 as pkg

    import __graft_entry__ as entry
    entry.build()
    lib, P = pkg.cabi.lib(), pkg.cabi.SetProblem
    fake = 256

    def prob(Q=900, n=10, **kw):
        d = dict(logits=fake, boxes=fake, gt_boxes=fake, gt_labels=fake, src=fake, tgt=fake, grad_logits=fake, grad_boxes=fake,
                 logit_stride=91, box_stride=4, num_queries=Q, num_gt=n, num_pairs=n, output=0)
        d.update(kw)
        return P(**d)

    def match(*ps, count=None):
        tab = (P * max(len(ps), 1))(*ps)
        return lib.sdetr_set_match(tab, len(ps) if count is None else count, 91, 2.0, 5.0, 2.0, 0.25, 2.0, fake, fake, 1 << 40,
                                   None)

    assert match(prob(logits=None)) == -1 and b"null pointer" in lib.sdetr_last_error()
    assert match(prob(gt_boxes=None)) == -1 and b"gt_boxes" in lib.sdetr_last_error()
    assert match(prob(src=None)) == -1
    assert match(prob(Q=100, n=101)) == -2 and b"n > Q" in lib.sdetr_last_error()
    assert match(prob(Q=4097, n=5)) == -2 and b"at most 4096" in lib.sdetr_last_error()
    assert match(prob(Q=0, n=0)) == -1
    assert match(prob(logit_stride=90)) == -1 and b"strides" in lib.sdetr_last_error()
    assert match(prob(), count=-1) == -1 and b"problems" in lib.sdetr_last_error()
    assert match(prob(), count=129) == -1
    tab = (P * 1)(prob())
    assert lib.sdetr_set_match(tab, 1, 91, 2.0, 5.0, 2.0, 0.25, 2.0, None, fake, 1 << 40, None) == -1  # status
    assert lib.sdetr_set_match(tab, 1, 91, 2.0, 5.0, 2.0, 0.25, 2.0, fake, fake, 10, None) == -4  # workspace
    assert lib.sdetr_set_match_workspace_floats(tab, 1) == 900 * 10
    assert lib.sdetr_set_assign(tab, 1, fake, 10, fake, None) == -1 and b"cost holds" in lib.sdetr_last_error()
    assert lib.sdetr_set_assign((P * 1)(prob(Q=8, n=9)), 1, fake, 1 << 40, fake, None) == -2
    # loss: output index, pair buffers, gradient buffers, loss pointer
    assert lib.sdetr_set_loss_forward(tab, 1, 0, 91, 0.25, 2.0, None, 1.0, None, fake, 1 << 40, fake, None) == -1
    assert lib.sdetr_set_loss_forward((P * 1)(prob(output=3)), 1, 2, 91, 0.25, 2.0, None, 1.0, None, fake, 1 << 40, fake,
                                      None) == -1 and b"names output 3" in lib.sdetr_last_error()
    assert lib.sdetr_set_loss_forward(tab, 1, 1, 91, 0.25, 2.0, None, 1.0, None, fake, 1 << 40, None, None) == -1
    assert lib.sdetr_set_loss_forward(tab, 1, 1, 91, 0.25, 2.0, None, 1.0, None, fake, 3, fake, None) == -4
    assert lib.sdetr_set_loss_workspace_floats(tab, 1) == 3 * (900 // 32 + 1)
    assert lib.sdetr_set_loss_backward((P * 1)(prob(grad_boxes=None)), 1, 1, 91, 0.25, 2.0, None, 1.0, None, fake, None) == -1
    assert lib.sdetr_set_loss_backward(tab, 1, 1, 91, 0.25, 2.0, None, 1.0, None, None, None) == -1
    assert lib.sdetr_set_loss_backward((P * 1)(prob(src=None)), 1, 1, 91, 0.25, 2.0, None, 1.0, None, fake, None) == -1


# ---- GPU -------------------------------------------------------------------------------------------------------------------------
def _pkg():
    import salience_detr_b200 as pkg
    return pkg


def _cuda_targets(targets):
    return [{"boxes": t["boxes"].cuda(), "labels": t["labels"].cuda()} for t in targets]


def _cuda_outputs(outputs, requires_grad=True):
    new = osc.to_dtype(outputs, torch.float32)
    leaves = []

    def mv(d):
        out = {k: v.cuda().requires_grad_(requires_grad) for k, v in d.items() if torch.is_tensor(v)}
        leaves.append(out)
        return out
    res = mv(new)
    if "aux_outputs" in new:
        res["aux_outputs"] = [mv(a) for a in new["aux_outputs"]]
    if "enc_outputs" in new:
        res["enc_outputs"] = mv(new["enc_outputs"])
    return res


def _criterion(K, binary):
    pkg = _pkg()
    c = osc.CONFIG
    m = pkg.HungarianMatcher(c["cost_class"], c["cost_bbox"], c["cost_giou"], c["alpha"], c["gamma"])
    return pkg.HybridSetCriterion(K, m, {}, alpha=c["alpha"], gamma=c["gamma"], two_stage_binary_cls=binary)


def _assign_problems(sizes, cost_fn, seed):
    pkg = _pkg()
    g = torch.Generator().manual_seed(seed)
    mats = [cost_fn(g, n, Q) for n, Q in sizes]  # (n, Q): rows gts, columns queries
    counts = [n for n, _ in sizes]
    pairs = torch.empty(2, max(sum(counts), 1), dtype=torch.int64, device="cuda")
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(int)
    structs = [pkg.cabi.SetProblem(src=pairs[0, o:].data_ptr(), tgt=pairs[1, o:].data_ptr(), num_queries=Q, num_gt=n)
               for (n, Q), o in zip(sizes, offs)]
    cost = torch.cat([m.reshape(-1) for m in mats]).cuda()
    status = torch.full((len(sizes),), -1, dtype=torch.int32, device="cuda")
    pkg.cabi.set_assign(structs, cost, status)
    torch.cuda.synchronize()
    return mats, [(pairs[0, o:o + n].cpu(), pairs[1, o:o + n].cpu()) for o, n in zip(offs, counts)], status.cpu()


SOLVER_SIZES = [(n, Q) for n in (0, 1, 2, 7, 30, 100, 300) for Q in sorted({max(n, 1), 300, 900, 4096}) if Q >= n]


@gpu
def test_solver_matches_scipy_on_tie_free_costs():
    sp = pytest.importorskip("scipy.optimize")
    mats, got, status = _assign_problems(SOLVER_SIZES, lambda g, n, Q: torch.rand(n, Q, generator=g) * 10 - 3, 5)
    assert torch.equal(status, torch.zeros_like(status))
    for (n, Q), m, (src, tgt) in zip(SOLVER_SIZES, mats, got):
        r, c = sp.linear_sum_assignment(m.t().double().numpy())
        assert np.array_equal(src.numpy(), r) and np.array_equal(tgt.numpy(), c), (n, Q)


@gpu
def test_solver_reaches_the_optimum_with_ties():
    sp = pytest.importorskip("scipy.optimize")
    mats, got, status = _assign_problems(SOLVER_SIZES, lambda g, n, Q: torch.randint(0, 4, (n, Q), generator=g).float(), 6)
    assert torch.equal(status, torch.zeros_like(status))
    for (n, Q), m, (src, tgt) in zip(SOLVER_SIZES, mats, got):
        r, c = sp.linear_sum_assignment(m.t().double().numpy())
        assert len(src) == n and bool((src[1:] > src[:-1]).all()) and sorted(tgt.tolist()) == list(range(n)), (n, Q)
        assert float(m.t().double()[src, tgt].sum()) == float(m.t().double().numpy()[r, c].sum()), (n, Q)


@gpu
def test_cost_kernel_matches_oracle_cost():
    pkg = _pkg()
    _, cfg, outputs, targets, _ = fixture("c2")
    tg = _cuda_targets(targets)
    out = _cuda_outputs(outputs, False)
    structs, want = [], []
    pairs = torch.empty(2, 6 * max(cfg["gt_counts"]), dtype=torch.int64, device="cuda")
    off = 0
    for o in [out] + out["aux_outputs"][:1] + [out["enc_outputs"]]:
        for i, t in enumerate(tg):
            lg, bx = o["pred_logits"][i], o["pred_boxes"][i]
            n = t["boxes"].shape[0]
            structs.append(pkg.cabi.SetProblem(logits=lg.data_ptr(), boxes=bx.data_ptr(), gt_boxes=t["boxes"].data_ptr(),
                                               gt_labels=t["labels"].data_ptr(), src=pairs[0, off:].data_ptr(),
                                               tgt=pairs[1, off:].data_ptr(),
                                               logit_stride=lg.stride(0), box_stride=bx.stride(0), num_queries=lg.shape[0],
                                               num_gt=n))
            off += n  # each problem writes its own index slots
            want.append(osc.cost_matrix(lg.cpu(), bx.cpu(), targets[i]["boxes"], targets[i]["labels"]).t())
    status = torch.empty(len(structs), dtype=torch.int32, device="cuda")
    c = osc.CONFIG
    ws = pkg.cabi.set_match(structs, cfg["K"], c["cost_class"], c["cost_bbox"], c["cost_giou"], c["alpha"], c["gamma"], status).cpu()
    off = 0
    for w in want:
        got = ws[off:off + w.numel()].view_as(w)
        off += w.numel()
        if w.numel():
            assert (got - w).abs().max() <= 1e-5 * w.abs().max()


def _run_criterion(name):
    z, cfg, outputs, targets, dn = fixture(name)
    crit = _criterion(cfg["K"], cfg["binary"])
    tg = _cuda_targets(targets)
    out = _cuda_outputs(outputs)
    losses = crit(out, tg)
    dl = dn_out = None
    if dn is not None:
        dn_out = _cuda_outputs(dn)
        ind = [(s.cuda(), t.cuda()) for s, t in osc.dn_indices(targets, int(z["dn.groups"]), int(z["dn.max_gt"]))]
        dl = crit.calculate_loss(dn_out, tg, num_boxes=osc.num_boxes_of(targets) * int(z["dn.groups"]), indices=ind)
    return z, cfg, crit, out, tg, losses, dn_out, dl


@gpu
@pytest.mark.parametrize("name", ["small", "c2"])
def test_criterion_matches_reference_fixture(name):
    z, cfg, crit, out, tg, losses, dn_out, dl = _run_criterion(name)
    # indices: the matcher is deterministic, so the criterion's own call matches these
    for suf, o in osc.flat_outputs(out):
        labels = [torch.zeros_like(t["labels"]) if suf == "_enc" and cfg["binary"] else t["labels"] for t in tg]
        ind, status = crit.matcher.match([(o["pred_logits"][i], o["pred_boxes"][i], t["boxes"], lb)
                                          for i, (t, lb) in enumerate(zip(tg, labels))])
        assert not status.any()
        for i, (s, t) in enumerate(ind):
            assert np.array_equal(s.cpu().numpy(), z[f"src{suf}_{i}"]) and np.array_equal(t.cpu().numpy(), z[f"tgt{suf}_{i}"])
    assert sorted(losses) == sorted(k[5:] for k in z.files if k.startswith("loss."))
    for k, v in losses.items():
        assert rel(v, z["loss." + k]) < 1e-5, (k, float(v), float(z["loss." + k]))
    total = sum(losses.values())
    if dl is not None:
        for k, v in dl.items():
            assert rel(v, z["dn." + k]) < 1e-5, k
        total = total + sum(dl.values())
    total.backward()
    for suf, o in osc.flat_outputs(out):
        check_grads(z, suf, (o["pred_logits"].grad.cpu().numpy(), o["pred_boxes"].grad.cpu().numpy()), 1e-5)
    if dl is not None:
        assert grad_err(dn_out["pred_logits"].grad.cpu().numpy(), z["dn.gl"]) < 1e-5
        assert grad_err(dn_out["pred_boxes"].grad.cpu().numpy(), z["dn.gb"]) < 1e-5


def _step(crit, out, tg):
    losses = crit(out, tg)
    base = losses["loss_class"]._base
    base.backward(torch.ones_like(base))
    return base


@gpu
def test_no_host_sync_and_bit_reproducible():
    z, cfg, outputs, targets, dn = fixture("c2")
    crit = _criterion(cfg["K"], cfg["binary"])
    tg = _cuda_targets(targets)
    runs = []
    for _ in range(2):
        out = _cuda_outputs(outputs)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = _step(crit, out, tg)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        runs.append([loss] + [t.grad for _, o in osc.flat_outputs(out) for t in (o["pred_logits"], o["pred_boxes"])])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@gpu
def test_launches_per_step_do_not_grow_with_outputs():
    from torch.profiler import ProfilerActivity, profile

    pkg = _pkg()
    counts = {}
    for num_aux in (0, 5):
        outputs, targets, _ = osc.synthetic_case(3, 2, 900, 91, (30, 7), num_aux, 850)
        crit = _criterion(91, False)
        tg = _cuda_targets(targets)
        out = _cuda_outputs(outputs)
        _step(crit, out, tg)
        out = _cuda_outputs(outputs)
        torch.cuda.synchronize()
        n0 = pkg.cabi.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _step(crit, out, tg)
            torch.cuda.synchronize()
        ours = pkg.cabi.launch_count() - n0
        kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        counts[num_aux] = (ours, len(kernels))
        print(f"outputs {num_aux + 2}: {ours} sdetr launches, {len(kernels)} GPU kernels/copies per forward + backward")
    assert counts[0] == counts[5]
    assert counts[5][0] == 4 and counts[5][1] <= 12


@gpu
def test_graph_capture_replays_bit_identically():
    _, cfg, outputs, targets, _ = fixture("small")
    crit = _criterion(cfg["K"], cfg["binary"])
    tg = _cuda_targets(targets)
    out = _cuda_outputs(outputs)
    leaves = [t for _, o in osc.flat_outputs(out) for t in (o["pred_logits"], o["pred_boxes"])]

    def step():
        for t in leaves:
            t.grad = None
        loss = _step(crit, out, tg)
        return [loss] + [t.grad for t in leaves]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for seed in (11, 12):  # new predictions and targets (same gt counts) copied into the static inputs
        new_out, new_tg, _ = osc.synthetic_case(seed, cfg["bs"], cfg["Q"], cfg["K"], cfg["gt_counts"], cfg["num_aux"],
                                                cfg["enc_q"])
        with torch.no_grad():
            for (_, o), (_, n) in zip(osc.flat_outputs(out), osc.flat_outputs(new_out)):
                o["pred_logits"].copy_(n["pred_logits"])
                o["pred_boxes"].copy_(n["pred_boxes"])
            for t, n in zip(tg, new_tg):
                t["boxes"].copy_(n["boxes"])
                t["labels"].copy_(n["labels"])
        graph.replay()
        got = [t.clone() for t in static]
        eager = step()
        for a, b in zip(got, eager):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@gpu
def test_nonfinite_input_gives_nan_without_sync_and_matcher_raises():
    _, cfg, outputs, targets, _ = fixture("small")
    crit = _criterion(cfg["K"], cfg["binary"])
    tg = _cuda_targets(targets)
    outputs["aux_outputs"][0]["pred_boxes"][1, 3, 0] = float("nan")  # the L1 cost of query 3 is NaN for every gt
    out = _cuda_outputs(outputs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = crit(out, tg)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(torch.isnan(losses[k + "_0"]) for k in osc.KEYS)
    assert all(torch.isfinite(losses[k]) and torch.isfinite(losses[k + "_enc"]) for k in osc.KEYS)
    o = out["aux_outputs"][0]
    with pytest.raises(ValueError):
        crit.matcher(o["pred_boxes"][1], o["pred_logits"][1], tg[1]["boxes"], tg[1]["labels"])
    src, tgt = crit.matcher(o["pred_boxes"][0], o["pred_logits"][0], tg[0]["boxes"], tg[0]["labels"])
    assert src.is_cuda and src.dtype == torch.int64 and len(src) == len(targets[0]["labels"])


@gpu
def test_cpu_inputs_raise():
    _, cfg, outputs, targets, _ = fixture("small")
    crit = _criterion(cfg["K"], cfg["binary"])
    with pytest.raises(RuntimeError):
        crit(outputs, targets)


@gpu
def test_label_out_of_range_gives_nan_and_matcher_raises():
    _, cfg, outputs, targets, _ = fixture("small")
    crit = _criterion(cfg["K"], cfg["binary"])
    tg = _cuda_targets(targets)
    tg[0]["labels"][2] = cfg["K"]  # one past the last class: an IndexError in the reference
    out = _cuda_outputs(outputs)
    ind, status = crit.matcher.match([(out["pred_logits"][i], out["pred_boxes"][i], t["boxes"], t["labels"])
                                      for i, t in enumerate(tg)])
    assert status.tolist() == [1, 0]
    losses = crit(out, tg)
    assert all(torch.isnan(losses[k]) and torch.isnan(losses[k + "_0"]) for k in osc.KEYS)
    assert all(torch.isfinite(losses[k + "_enc"]) for k in osc.KEYS)  # two_stage_binary_cls: every label is 0
    dn = crit.calculate_loss(out, tg, 1.0, indices=[(torch.arange(3, device="cuda"), torch.arange(3, device="cuda")),
                                                    (torch.arange(2, device="cuda"), torch.arange(2, device="cuda"))])
    assert all(torch.isnan(v) for v in dn.values())
    with pytest.raises(IndexError):
        crit.matcher(out["pred_boxes"][0], out["pred_logits"][0], tg[0]["boxes"], tg[0]["labels"])


@gpu
def test_more_problems_than_one_call_holds():
    """bs = 20 with 7 outputs: 140 (output, image) problems, split over two loss calls of whole outputs."""
    outputs, targets, _ = osc.synthetic_case(21, 20, 60, 5, [2, 0, 3, 1] * 5, 5, 40)
    crit = _criterion(5, False)
    tg = _cuda_targets(targets)
    out = _cuda_outputs(outputs)
    losses = crit(out, tg)
    idx = {}
    for suf, o in osc.flat_outputs(out):
        ind, status = crit.matcher.match([(o["pred_logits"][i], o["pred_boxes"][i], t["boxes"], t["labels"])
                                          for i, t in enumerate(tg)])
        assert not status.any()
        idx[suf] = [(s.cpu(), t.cpu()) for s, t in ind]
    sum(losses.values()).backward()
    out64 = osc.to_dtype(outputs, torch.float64, requires_grad=True)
    want, _ = osc.criterion(out64, [dict(t, boxes=t["boxes"].double()) for t in targets], indices=idx)
    sum(want.values()).backward()
    for k, v in want.items():
        assert rel(losses[k], v) < 1e-5, k
    for (suf, o), (_, o64) in zip(osc.flat_outputs(out), osc.flat_outputs(out64)):
        for key in ("pred_logits", "pred_boxes"):
            assert grad_err(o[key].grad.cpu().numpy(), o64[key].grad.numpy()) < 1e-5, (suf, key)


@gpu
def test_in_place_change_before_backward_is_an_error():
    _, cfg, outputs, targets, _ = fixture("small")
    crit = _criterion(cfg["K"], cfg["binary"])
    out = _cuda_outputs(outputs, False)
    logits = out["pred_logits"].clone().requires_grad_(True)
    x = logits * 1.0
    losses = crit(dict(out, pred_logits=x), _cuda_targets(targets))
    with torch.no_grad():
        x.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        losses["loss_class"].backward()


# ---- end to end: the decoder's stacked outputs through the criterion, gradients against a float64 twin -----------------------
def _training_gradients():
    import test_training_gradients as ttg
    return ttg


def _split_like_dn_post_process(cls, box, pad):
    """DNDETRDetector.dn_post_process + DETRDetector._set_aux_loss: views of the stacked (layers, b, pad + Q, .) outputs."""
    def outs(c, b):
        return {"pred_logits": c[-1], "pred_boxes": b[-1],
                "aux_outputs": [{"pred_logits": x, "pred_boxes": y} for x, y in zip(c[:-1], b[:-1])]}
    matched = outs(cls[:, :, pad:], box[:, :, pad:])
    return matched, (outs(cls[:, :, :pad], box[:, :, :pad]) if pad else None)


def _decoder_loss_grads(decoder, kw, dtype, loss_fn):
    q = kw["query"].detach().to(dtype).requires_grad_(True)
    v = kw["value"].detach().to(dtype).requires_grad_(True)
    args = dict(kw, query=q, value=v, reference_points=kw["reference_points"].to(dtype), valid_ratios=kw["valid_ratios"].to(dtype))
    cls, box = decoder(**args)
    loss_fn(cls, box).backward()
    out = {n: p.grad for n, p in decoder.named_parameters() if p.grad is not None}
    out.update(value=v.grad, query=q.grad)
    return out


@gpu
@pytest.mark.parametrize("mode", ["atomic", "deterministic"])
@pytest.mark.parametrize("denoising", [False, True])
def test_decoder_training_with_set_criterion_vs_float64(denoising, mode):
    """The setup of test_training_gradients.test_decoder_training_vs_float64 (HALF geometry: 3 layers, 300 queries, with and
    without 20 denoising queries and their mask) with this HybridSetCriterion in place of the linear functional: matched
    outputs and aux_outputs, plus the denoising outputs through calculate_loss(indices=...), all read in place from the
    decoder's stacked outputs.  Every decoder parameter gradient, value.grad and query.grad against a float64 twin that runs
    the oracle criterion with OUR indices (so near-ties cannot make the two sides match differently)."""
    import salience_detr_b200 as pkg
    from oracle import make_golden as mg
    from oracle import oracle as orc
    ttg = _training_gradients()
    tdh = ttg._decoder_half()
    g, shapes = tdh._golden(False)
    ours = tdh._ours(pkg, shapes).train()
    b = g["reference_points"].shape[0]
    nv = int(g["key_padding_mask"].shape[1])
    dev = ttg.DEV
    kw = dict(query=ours.tgt_embed.weight.detach().expand(b, -1, -1).contiguous(),
              value=orc.seeded_memory((b, nv, mg.HALF["embed_dim"]), mg.HALF_VALUE_SEED).to(dev),
              key_padding_mask=g["key_padding_mask"].to(dev), reference_points=g["reference_points"].to(dev),
              spatial_shapes=g["spatial_shapes"].to(dev), level_start_index=g["level_start_index"].to(dev),
              valid_ratios=g["valid_ratios"].to(dev), attn_mask=None)
    pad, gt_counts = 0, (5, 3)[:b] + (4,) * max(b - 2, 0)
    groups, max_gt = 20 // max(gt_counts), max(gt_counts)
    if denoising:
        dn_q, dn_b, mask = orc.denoising_queries(b, kw["query"].shape[1], mg.HALF["embed_dim"])
        pad = dn_q.shape[1]
        assert pad == groups * max_gt
        kw.update(query=torch.cat([dn_q.to(dev), kw["query"]], 1),
                  reference_points=torch.cat([dn_b.to(dev), kw["reference_points"]], 1), attn_mask=mask.to(dev))
    K = mg.HALF["num_classes"]
    gen = torch.Generator().manual_seed(13)
    targets = [{"boxes": osc.random_boxes(gen, n).to(dev), "labels": torch.randint(0, K, (n,), generator=gen).to(dev)}
               for n in gt_counts]
    dn_idx = [(s.to(dev), t.to(dev)) for s, t in osc.dn_indices(targets, groups, max_gt)]
    crit = _criterion(K, False)
    nb = pkg.set_criterion.num_boxes_of(targets)
    used = {}

    def our_loss(cls, box):
        matched, dn = _split_like_dn_post_process(cls, box, pad)
        with torch.no_grad():  # the indices the criterion computes inside (the matcher is deterministic), for the twins
            for suf, o in osc.flat_outputs(matched):
                ind, status = crit.matcher.match([(o["pred_logits"][i], o["pred_boxes"][i], t["boxes"], t["labels"])
                                                  for i, t in enumerate(targets)])
                assert not status.any()
                used[suf] = [(s.clone(), t.clone()) for s, t in ind]
        losses = crit(matched, targets)
        for j, o in enumerate([dn] + dn["aux_outputs"] if dn else []):
            losses.update({f"{k}_dn_{j}": v for k, v in crit.calculate_loss(o, targets, nb * groups, indices=dn_idx).items()})
        return sum(losses.values())

    def twin_loss(dtype):
        def fn(cls, box):
            matched, dn = _split_like_dn_post_process(cls, box, pad)
            tg = [dict(t, boxes=t["boxes"].to(dtype)) for t in targets]
            losses, _ = osc.criterion(matched, tg, indices=used)
            for j, o in enumerate([dn] + dn["aux_outputs"] if dn else []):
                for k, v in osc.calculate_loss(o["pred_logits"], o["pred_boxes"], tg, nb * groups, dn_idx).items():
                    losses[f"{k}_dn_{j}"] = v
            return sum(losses.values())
        return fn

    with ttg._backward_mode(mode):
        got = _decoder_loss_grads(ours.decoder, kw, torch.float32, our_loss)
    want = _decoder_loss_grads(ttg._decoder_twin(ours.decoder, torch.float64), kw, torch.float64, twin_loss(torch.float64))
    plain = _decoder_loss_grads(ttg._decoder_twin(ours.decoder, torch.float32), kw, torch.float32, twin_loss(torch.float32))
    ttg._assert_within(f"decoder + set criterion dn={denoising} {mode}", got, want, plain)
