"""PostProcess on the GPU (salience-detr_b200/postprocess.py, csrc/postprocess.cu) against the fixture made from the unmodified
reference (tests/golden/postprocess.npz, tools/make_postprocess_golden.py) and the plain-torch restatement below, which the CPU
tests pin to that fixture."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from tools import make_postprocess_golden as mpg

gpu = pytest.mark.gpu
NAMES = list(mpg.CASES)
DEV = "cuda:0"


def _pkg():
    import salience_detr_b200 as pkg
    return pkg


# ---- the restatement ---------------------------------------------------------------------------------------------------------
def greedy_nms(boxes, thr):
    """Sequential greedy NMS over the rows of boxes (k, 4) xyxy in row order, torchvision's IoU with every operation rounded
    separately -> keep mask (k,)."""
    x1, y1, x2, y2 = boxes.unbind(-1)
    area = (x2 - x1) * (y2 - y1)
    w = (torch.minimum(x2[:, None], x2[None]) - torch.maximum(x1[:, None], x1[None])).clamp(min=0)
    h = (torch.minimum(y2[:, None], y2[None]) - torch.maximum(y1[:, None], y1[None])).clamp(min=0)
    inter = w * h
    over = (inter / (area[:, None] + area[None] - inter) > thr).cpu().numpy()
    supp = np.zeros(len(boxes), dtype=bool)
    for i in range(len(boxes)):
        if not supp[i]:
            supp[i + 1:] |= over[i, i + 1:]
    return torch.from_numpy(~supp).to(boxes.device)


def restate(logits, boxes, sizes, k, nms=-1, conf=-1):
    """PostProcess.forward (post_process.py:21-74) in plain torch, ties in the canonical order (stable descending sort) and
    NMS visiting the boxes in that order.  -> per image (scores, labels, boxes, flat indices)."""
    b, Q, K = logits.shape
    scores, idx = torch.sort(logits.sigmoid().reshape(b, -1), dim=1, descending=True, stable=True)
    scores, idx = scores[:, :k], idx[:, :k]
    labels = idx % K
    cx, cy, w, h = boxes.unbind(-1)
    xyxy = torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], dim=-1)
    xyxy = torch.gather(xyxy, 1, torch.div(idx, K, rounding_mode="trunc").unsqueeze(-1).repeat(1, 1, 4))
    img_h, img_w = sizes.unbind(1)
    xyxy = xyxy * torch.stack([img_w, img_h, img_w, img_h], dim=1)[:, None, :]
    out = []
    for i in range(b):
        keep = torch.ones(k, dtype=torch.bool, device=logits.device)
        if conf > 0:
            keep &= scores[i] > conf
        if nms > 0:
            keep &= greedy_nms(xyxy[i], nms)
        out.append((scores[i][keep], labels[i][keep], xyxy[i][keep], idx[i][keep]))
    return out


def bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def entries(scores, labels, boxes):
    """score bits -> list of (label, box bits) in order"""
    groups = {}
    for s, lab, bx in zip(bits(scores).tolist(), labels.cpu().tolist(), bits(boxes).tolist()):
        groups.setdefault(s, []).append((lab, tuple(bx)))
    return groups


def assert_equal_up_to_ties(want, got, pool):
    """Scores position for position; within each group of equal scores the (label, box) entries as sets.  A group cut by k
    (fewer entries than `pool`, the whole candidate list, has with that score) only needs entries from the pool."""
    assert same_bits(want[0], got[0])
    gw, gg, gp = entries(*want[:3]), entries(*got[:3]), entries(*pool[:3])
    for s, ew in gw.items():
        if len(gp[s]) == len(ew):
            assert sorted(ew) == sorted(gg[s]), s
        else:
            assert set(ew) <= set(gp[s]) and set(gg[s]) <= set(gp[s]), s


def fixture():
    return np.load(os.path.join(GOLDEN, "postprocess.npz"))


def case(z, name):
    outputs, sizes = mpg.case_inputs(name, int(z["seed"]) + NAMES.index(name))
    b, Q, K, k, nms, conf, _ = mpg.CASES[name]
    return outputs, sizes, k, nms, conf


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_restatement_reproduces_fixture(name):
    z = fixture()
    outputs, sizes, k, nms, conf = case(z, name)
    logits, boxes = outputs["pred_logits"], outputs["pred_boxes"]
    got = restate(logits, boxes, sizes, k, nms, conf)
    pool = restate(logits, boxes, sizes, logits.shape[1] * logits.shape[2])
    for i, g in enumerate(got):
        want = tuple(torch.from_numpy(z[f"{name}.{i}.{key}"]) for key in ("scores", "labels", "boxes"))
        assert want[1].dtype == torch.int64 and want[2].dtype == torch.float32
        assert_equal_up_to_ties(want, g, pool[i])


def test_errors_on_the_host():
    """The reference's assertions and TypeError, and CPU tensors, before anything reaches the library."""
    pkg = _pkg()
    outputs, sizes = mpg.case_inputs("q300_c80", 0)
    with pytest.raises(AssertionError):
        pkg.PostProcess(100)(outputs, sizes[:1])
    with pytest.raises(AssertionError):
        pkg.PostProcess(100)(outputs, torch.ones(2, 3, dtype=torch.int64))
    with pytest.raises(TypeError):
        pkg.PostProcess(100, nms_iou_threshold=0.5)(outputs, sizes)
    with pytest.raises(RuntimeError, match="CUDA"):
        pkg.PostProcess(100)(outputs, sizes)
    m = pkg.PostProcess(300, 0.7, 0.2)
    assert (m.select_box_nums_for_evaluation, m.nms_iou_threshold, m.confidence_score) == (300, 0.7, 0.2)


def test_cabi_rejects_malformed_arguments():
    """Argument checks run on the host before any CUDA call."""
    import __graft_entry__ as entry
    entry.build()
    lib = _pkg().cabi.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ws = lib.sdetr_postprocess_workspace(2, 900, 91)
    assert ws == 2 * 900 * 91 * 4

    def call(logits=p, sizes=p, dtype=0, b=2, Q=900, K=91, k=100, conf=-1.0, iou=-1.0, count=p, wsb=ws):
        return lib.sdetr_postprocess(logits, 91 * 900, 91, p, 3600, 4, sizes, dtype, b, Q, K, k, conf, iou, p, p, p, count, p,
                                     wsb, None)

    for kw, code, msg in [(dict(logits=None), -1, b"null pointer"), (dict(sizes=None), -1, b"null pointer"),
                          (dict(count=None, conf=0.3), -1, b"count"), (dict(count=None, iou=0.5), -1, b"count"),
                          (dict(k=0), -1, b"k=0"), (dict(k=-3), -1, b"k=-3"), (dict(Q=10, K=9, k=91), -1, b"k=91"),
                          (dict(k=4097), -2, b"at most 4096"), (dict(dtype=3), -1, b"dtype code 3"),
                          (dict(b=0), -1, b"bad sizes"), (dict(Q=50000, K=50000, k=10), -2, b"2^31"),
                          (dict(wsb=ws - 1), -4, b"workspace")]:
        rc = call(**kw)
        assert rc == code and msg in lib.sdetr_last_error(), (kw, rc, lib.sdetr_last_error())


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
SHAPES = [(900, 91), (300, 80), (1100, 91)]
KS = [1, 100, 300, 4096]


def gpu_inputs(b, Q, K, seed, ties=False, sizes_dtype=torch.int64):
    g = torch.Generator().manual_seed(seed)
    if ties:  # quantised logits: heavy exact ties, plus +-inf and NaN
        logits = torch.randint(-12, 5, (b, Q, K), generator=g).float() * 0.75
        flat = logits.view(b, -1)
        for i in range(b):
            pos = torch.randperm(Q * K, generator=g)[:6]
            flat[i, pos[:2]] = float("inf")
            flat[i, pos[2:4]] = float("-inf")
            flat[i, pos[4:]] = float("nan")
    else:
        logits = torch.randn(b, Q, K, generator=g) * 1.5 - 4.5
    boxes = torch.cat([torch.rand(b, Q, 2, generator=g) * 0.9 + 0.05, torch.rand(b, Q, 2, generator=g) * 0.4 + 0.02], -1)
    sizes = torch.stack([torch.randint(300, 1334, (b,), generator=g), torch.randint(300, 1334, (b,), generator=g)], 1)
    return logits.to(DEV), boxes.to(DEV), sizes.to(sizes_dtype).to(DEV)


def run(logits, boxes, sizes, k, nms=-1, conf=-1):
    return _pkg().PostProcess(k, nms, conf)({"pred_logits": logits, "pred_boxes": boxes}, sizes)


def assert_same(res, want):
    assert len(res) == len(want)
    for r, (s, lab, bx, _) in zip(res, want):
        assert r["labels"].dtype == torch.int64 and r["scores"].dtype == torch.float32 and r["boxes"].dtype == torch.float32
        assert same_bits(r["scores"], s) and torch.equal(r["labels"], lab) and same_bits(r["boxes"], bx)


@gpu
@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("b", [1, 2, 8])
@pytest.mark.parametrize("shape", SHAPES)
def test_topk_decode_bit_exact(shape, b, k, ties):
    """Scores == torch.sigmoid on CUDA, indices == the stable sort on CUDA (ties, NaN, +-inf), boxes == the torch chain."""
    Q, K = shape
    logits, boxes, sizes = gpu_inputs(b, Q, K, seed=Q + b + k + ties, ties=ties)
    assert_same(run(logits, boxes, sizes, k), restate(logits, boxes, sizes, k))


@gpu
@pytest.mark.parametrize("sizes_dtype", [torch.int64, torch.int32, torch.float32])
def test_target_size_dtypes(sizes_dtype):
    logits, boxes, sizes = gpu_inputs(2, 900, 91, seed=5, sizes_dtype=sizes_dtype)
    if sizes_dtype == torch.float32:
        sizes = sizes + 0.37  # non-integer sizes
    assert_same(run(logits, boxes, sizes, 300), restate(logits, boxes, sizes, 300))


@gpu
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("b", [1, 2, 8])
@pytest.mark.parametrize("shape", SHAPES)
def test_filters_match_torchvision(shape, b, k):
    """Confidence filter AND torchvision.ops.nms on CUDA, per image, on tie-free random scores and boxes."""
    import torchvision
    Q, K = shape
    logits, boxes, sizes = gpu_inputs(b, Q, K, seed=7 * Q + b + k)
    for nms, conf in [(0.5, 0.3), (0.7, 0.05), (-1, 0.4)]:
        got = run(logits, boxes, sizes, k, nms, conf)
        full = restate(logits, boxes, sizes, k)
        for r, (s, lab, bx, _) in zip(got, full):
            keep = s > conf
            if nms > 0:
                mask = torch.zeros_like(keep)
                mask[torchvision.ops.nms(bx, s, nms)] = True
                keep &= mask
            assert same_bits(r["scores"], s[keep]) and torch.equal(r["labels"], lab[keep]) and same_bits(r["boxes"], bx[keep])


@gpu
def test_iou_exactly_at_threshold_is_not_suppressed():
    # integer boxes on a 1 x 1 image: A = [0,0,3,1], B = [1,0,4,1] (IoU with A exactly 0.5), C = [0.5,0,3.5,1] (IoU 5/7 with A)
    logits = torch.tensor([[[3.0], [2.0], [1.0]]], device=DEV)
    boxes = torch.tensor([[[1.5, 0.5, 3.0, 1.0], [2.5, 0.5, 3.0, 1.0], [2.0, 0.5, 3.0, 1.0]]], device=DEV)
    sizes = torch.ones(1, 2, dtype=torch.int64, device=DEV)
    r = run(logits, boxes, sizes, 3, 0.5, 0.1)[0]
    assert r["boxes"].tolist() == [[0.0, 0.0, 3.0, 1.0], [1.0, 0.0, 4.0, 1.0]]
    assert len(run(logits, boxes, sizes, 3, 0.49, 0.1)[0]["scores"]) == 1


@gpu
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("shape", SHAPES)
def test_tied_scores_follow_sequential_greedy(shape, k):
    """With heavy score ties the kept list equals a sequential greedy loop in the canonical top-k order; integer-ish boxes so
    that IoUs tie too."""
    Q, K = shape
    logits, boxes, sizes = gpu_inputs(2, Q, K, seed=11 + k, ties=True)
    boxes = (boxes * 16).round() / 16
    for nms, conf in [(0.5, 0.01), (0.3, 0.2)]:
        assert_same(run(logits, boxes, sizes, k, nms, conf), restate(logits, boxes, sizes, k, nms, conf))


@gpu
@pytest.mark.parametrize("filters", [(-1, -1), (0.5, 0.3)])
def test_strided_query_slice(filters):
    """outputs_class[:, :, pad:, :] as dn_post_process leaves it: no copy, same result as the contiguous tensor.  One
    library launch, and the call's peak allocation is no larger than on the contiguous tensors: a copy of either slice
    would add at least the size of the smaller one (the boxes) while the call runs."""
    pad = 37
    logits, boxes, sizes = gpu_inputs(2, 900 + pad, 91, seed=3)
    ls, bs = logits[:, pad:, :], boxes[:, pad:, :]
    assert not ls.is_contiguous() and not bs.is_contiguous()
    lc, bc = ls.contiguous(), bs.contiguous()
    pkg = _pkg()

    def peak_and_launches(lg, bx):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base, n0 = torch.cuda.memory_allocated(), pkg.cabi.launch_count()
        out = run(lg, bx, sizes, 300, *filters)
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated() - base, pkg.cabi.launch_count() - n0

    want, peak_contiguous, _ = peak_and_launches(lc, bc)
    got, peak, launches = peak_and_launches(ls, bs)
    assert launches == 1
    assert peak <= peak_contiguous, (peak, peak_contiguous)
    for r, w in zip(got, want):
        assert all(same_bits(r[key], w[key]) for key in ("scores", "labels", "boxes"))


@gpu
def test_filters_off_one_launch_no_sync_graph():
    pkg = _pkg()
    logits, boxes, sizes = gpu_inputs(2, 900, 91, seed=9)
    m = pkg.PostProcess(300)
    outputs = {"pred_logits": logits, "pred_boxes": boxes}
    want = m(outputs, sizes)
    torch.cuda.synchronize()
    n0 = pkg.cabi.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = m(outputs, sizes)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert pkg.cabi.launch_count() - n0 == 1
    assert got[0]["scores"]._base is not None  # a view of the padded (b, k) buffer
    for r, w in zip(got, want):
        assert all(same_bits(r[key], w[key]) for key in ("scores", "labels", "boxes"))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m(outputs, sizes)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = m(outputs, sizes)
    logits.copy_(gpu_inputs(2, 900, 91, seed=10)[0])
    graph.replay()
    torch.cuda.synchronize()
    eager = m(outputs, sizes)
    for r, w in zip(cap, eager):
        assert all(same_bits(r[key], w[key]) for key in ("scores", "labels", "boxes"))


@gpu
def test_filters_on_one_launch():
    pkg = _pkg()
    logits, boxes, sizes = gpu_inputs(8, 900, 91, seed=12)
    torch.cuda.synchronize()
    n0 = pkg.cabi.launch_count()
    run(logits, boxes, sizes, 300, 0.5, 0.3)
    assert pkg.cabi.launch_count() - n0 == 1


@gpu
@pytest.mark.parametrize("filters", [(-1, -1), (0.5, 0.3)])
def test_repeatable(filters):
    logits, boxes, sizes = gpu_inputs(8, 900, 91, seed=13, ties=True)
    a, b = run(logits, boxes, sizes, 4096, *filters), run(logits, boxes, sizes, 4096, *filters)
    for r, w in zip(a, b):
        assert all(same_bits(r[key], w[key]) for key in ("scores", "labels", "boxes"))


@gpu
def test_errors_on_the_gpu():
    logits, boxes, sizes = gpu_inputs(2, 30, 10, seed=1)
    with pytest.raises(AssertionError):
        run(logits, boxes, sizes[:1], 10)
    with pytest.raises(AssertionError):
        run(logits, boxes, torch.ones(2, 3, dtype=torch.int64, device=DEV), 10)
    with pytest.raises(RuntimeError, match="out of range"):
        run(logits, boxes, sizes, 301)
    with pytest.raises(TypeError):
        run(logits, boxes, sizes, 10, 0.5, -1)
    with pytest.raises(RuntimeError, match="float32"):
        run(logits.half(), boxes, sizes, 10)
    with pytest.raises(RuntimeError, match="float64"):
        run(logits, boxes, sizes.double(), 10)
    big, bboxes, bsizes = gpu_inputs(1, 900, 91, seed=1)
    with pytest.raises(RuntimeError, match="4096"):
        run(big, bboxes, bsizes, 4097)
    with pytest.raises(RuntimeError, match="CUDA"):
        run(logits.cpu(), boxes.cpu(), sizes.cpu(), 10)


@gpu
def test_through_the_decoder():
    """The HALF-geometry SalienceTransformer (tests/test_decoder_half.py) in eval, then PostProcess(300): equal to the
    restatement on the same logits."""
    import test_decoder_half as tdh
    pkg = _pkg()
    _, shapes = tdh._golden(False)
    model = tdh._ours(pkg, shapes)
    feats, masks, pos = tdh._inputs(False)
    with torch.no_grad():
        out = model(feats, masks, pos, None, None, None)
    logits, boxes = out[0][-1], out[1][-1]
    sizes = torch.tensor([[480, 640], [427, 640]], device=DEV)[: logits.shape[0]]
    for filters in [(-1, -1), (0.5, 0.3)]:
        assert_same(run(logits, boxes, sizes, 300, *filters), restate(logits, boxes, sizes, 300, *filters))
