"""The salience filter (sdetr_salience_select) on each of its three code paths, and sdetr_topk_desc, against a plain torch
reference: at the shapes where the host switches paths, and on adversarial scores -- heavy ties, -0 mixed with +0, +-inf,
NaNs of both signs and several payloads, flat levels, padding fills equal to real scores.

The host picks a path from the level budgets k_l and, when a processing order is wanted, the size of the spatial-cell
histogram (`select_path` restates the rule):
1. rank merge: the winners fit in at most 32 slices of 2048 and the histogram has at most 12000 bins;
2. bitonic merge: otherwise, when K <= 16384 (one CTA sorts all K winners in shared memory);
3. LSD radix sorts through global memory: every other case.
Every GPU case checks under torch.profiler that the kernels of its predicted path ran."""
import time

import numpy as np
import pytest
import torch

from conftest import TINY_CFG
from oracle import oracle as orc

DEV = "cuda:0"
CELL_PX = 64
SLICE, MAX_LISTS, MAX_BINS, BITONIC_MAX = 2048, 32, 12000, 16384
CANONICAL_NAN = torch.tensor([0x7FFFFFFF], dtype=torch.int32).view(torch.float32)[0]


# ---- the reference -------------------------------------------------------------------------------------------------
def _score_min(x):
    """`x.min()` with the two edges torch leaves to the backend pinned the way the kernel computes them: a NaN propagates
    as the canonical NaN 0x7fffffff (torch's CPU min returns 0xffffffff, its CUDA min one of the inputs), and a minimum
    of +0 and -0 is -0 (torch returns whichever it meets first)."""
    if x.isnan().any():
        return CANONICAL_NAN.clone()
    m = x.min()
    if m == 0 and torch.signbit(x[x == 0]).any():
        return torch.tensor(-0.0)
    return m


def torch_salience_select(raw, mask, starts, sizes, k):
    """salience_transformer.py:146-168 on the CPU, with a stable sort in place of topk so that ties fall by ascending index.
    -> selected_inds (b, K) int64, selected_score (b, K), foreground_score (b, Nv).  No arithmetic: exact in fp32."""
    mins, scores, inds = [], [], []
    for s, n, kl in zip(starts, sizes, k):
        level = raw[:, s:s + n]
        m = _score_min(level)  # py:146 `score.min()` over the whole batch
        mins.append(m)
        filled = level.masked_fill(mask[:, s:s + n], m)
        v, i = torch.sort(filled, dim=1, descending=True, stable=True)  # py:150
        scores.append(v[:, :kl])
        inds.append(i[:, :kl] + s)  # py:151
    score, order = torch.sort(torch.cat(scores, 1), dim=1, descending=True, stable=True)  # py:156-157
    sel = torch.cat(inds, 1).gather(1, order)  # py:158
    fg = raw.masked_fill(mask, _score_min(torch.stack(mins)))  # py:167-168
    return sel, score, fg


# ---- the host's path rule --------------------------------------------------------------------------------------------
def select_path(shapes, k, strides, cell_px, want_order):
    """Which path sdetr_salience_select takes (0: K = 0, nothing beyond the foreground score)."""
    K = sum(k)
    if K == 0:
        return 0
    slices = sum(-(-kl // SLICE) for kl in k)
    bins = 0
    if want_order:
        cells_x = (max(w * s for (_, w), s in zip(shapes, strides)) + cell_px - 1) // cell_px + 1
        cells_y = (max(h * s for (h, _), s in zip(shapes, strides)) + cell_px - 1) // cell_px + 1
        bins = cells_y * cells_x * 8
    if slices <= MAX_LISTS and bins <= MAX_BINS:
        return 1
    return 2 if K <= BITONIC_MAX else 3


PATH_KERNELS = {
    0: set(),
    1: {"level_select_sort_kernel", "merge_rank_kernel"},
    2: {"level_select_kernel", "merge_bitonic_kernel"},
    3: {"level_sort_kernel", "merge_sort_kernel"},
}
ORDER_KERNEL = {1: {"tile_count_kernel"}, 2: set(), 3: {"tile_order_kernel"}}  # path 2 orders inside merge_bitonic
KERNEL_NAMES = {"level_min_kernel", "foreground_kernel", "topk_select_kernel", "topk_kernel", "order_prefix_kernel",
                *ORDER_KERNEL[1], *ORDER_KERNEL[3], *(n for v in PATH_KERNELS.values() for n in v)}


def expected_kernels(path, want_order):
    return {"level_min_kernel", "foreground_kernel"} | PATH_KERNELS[path] | (ORDER_KERNEL.get(path, set()) if want_order else set())


# ---- cases -----------------------------------------------------------------------------------------------------------
def _case(id, b, shapes, k, order, path, strides=None, pad=None, full=()):
    """pad[i]: the right-hand fraction of image i that is padding (every level); full: (image, level) pairs masked whole."""
    return dict(id=id, b=b, shapes=shapes, k=k, order=order, path=path,
                strides=strides or [8 * 2 ** l for l in range(len(shapes))], pad=pad, full=full)


BIG = [(400, 400), (200, 200)]            # 3200 px: 51 x 51 cells, 20 808 bins > 12 000
AT_BINS = [(232, 392), (116, 196)]        # 30 x 50 cells: exactly 12 000 bins
OVER_BINS = [(232, 393), (116, 197)]      # 30 x 51 cells: 12 240 bins
FOUR = [(90, 100), (45, 50), (23, 25), (12, 13)]
CASES = [
    # path 1: rank merge
    _case("p1_32_slices", 2, [(300, 300)], [32 * SLICE], False, 1, pad=[0.0, 0.3]),
    _case("p1_slice_edges", 3, FOUR, [2 * SLICE, SLICE + 1, 575, 1], True, 1, pad=[0.0, 0.2, 0.6], full=[(1, 2)]),
    _case("p1_k0_level_and_k_eq_size", 2, [(20, 30), (10, 15), (5, 8)], [0, 150, 40], True, 1, pad=[0.3, 0.0]),
    _case("p1_k0_level_unordered", 1, [(20, 30), (10, 15), (5, 8)], [300, 0, 7], False, 1),
    _case("p1_bins_12000", 2, AT_BINS, [6000, 3000], True, 1, pad=[0.0, 0.4], full=[(1, 1)]),
    _case("p1_five_levels", 2, [(60, 84), (30, 42), (15, 21), (8, 11), (4, 6)], [2016, 1008, 315, 88, 24], True, 1,
          strides=[4, 8, 16, 32, 64], pad=[0.1, 0.0]),
    _case("k_zero", 2, [(20, 30), (10, 15)], [0, 0], True, 0, pad=[0.0, 0.5]),
    # path 2: bitonic merge (the histogram is too large; K <= 16 384), N = next_pow2(K) below and above one CTA
    _case("p2_bins_12240", 2, OVER_BINS, [6000, 3000], True, 2, pad=[0.0, 0.4], full=[(1, 1)]),
    _case("p2_K1", 1, BIG, [1, 0], True, 2),
    _case("p2_K31", 3, BIG, [20, 11], True, 2, pad=[0.0, 0.1, 0.5], full=[(2, 1)]),
    _case("p2_K32", 2, BIG, [0, 32], True, 2, pad=[0.2, 0.0]),
    _case("p2_K480", 3, BIG, [320, 160], True, 2, pad=[0.0, 0.05, 0.3]),
    _case("p2_K1024", 2, BIG, [1000, 24], True, 2, pad=[0.0, 0.3], full=[(0, 1)]),
    _case("p2_K16384", 2, BIG, [12000, 4384], True, 2, pad=[0.1, 0.0]),
    # path 3: LSD radix sorts
    _case("p3_K16385", 2, BIG, [12000, 4385], True, 3, pad=[0.1, 0.0]),
    _case("p3_ordered", 3, BIG, [16000, 8000], True, 3, pad=[0.0, 0.2, 0.5], full=[(2, 1)]),
    _case("p3_33_slices", 2, [(300, 300)], [32 * SLICE + 1], False, 3, pad=[0.0, 0.3]),
    _case("p3_unordered", 2, [(300, 300)], [67500], False, 3, pad=[0.25, 0.0]),
]
KINDS = ["ties", "zeros", "inf", "nan", "flat"]
NAN_BITS = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF], dtype=np.uint32)  # quiet, negative, signalling, all ones


def make_scores(kind, b, sizes, g):
    """(b, sum(sizes)) scores of one adversarial kind; the levels are the column ranges of `sizes`."""
    nv = sum(sizes)
    q = ((torch.randn(b, nv, generator=g) * 2).round() / 2).clamp(-2, 2)  # nine values, -0 among them; the min recurs
    if kind == "ties":
        return q
    if kind == "zeros":  # -0 and +0 tie, and they are the level minimum
        return torch.tensor([-0.0, 0.0, 0.5, 1.0])[torch.randint(0, 4, (b, nv), generator=g)]
    r = torch.rand(b, nv, generator=g)
    if kind == "inf":
        q[r < 0.05] = float("inf")
        q[r > 0.95] = -float("inf")
        return q
    if kind == "nan":  # NaNs in every level but the last one: a NaN level minimum next to a finite one
        nan = torch.from_numpy(NAN_BITS.view(np.float32))[torch.randint(0, 4, (b, nv), generator=g)]
        hit = r < 0.04
        if len(sizes) > 1:
            hit[:, nv - sizes[-1]:] = False
        q[hit] = nan[hit]
        q[r > 0.98] = float("inf")
        return q
    if kind == "flat":  # the first level all equal, so also to its own padding fill
        q[:, :sizes[0]] = 0.75
        return q
    raise ValueError(kind)


def make_mask(case):
    shapes, b = case["shapes"], case["b"]
    parts = []
    for l, (h, w) in enumerate(shapes):
        m = torch.zeros(b, h, w, dtype=torch.bool)
        for i, frac in enumerate(case["pad"] or []):
            m[i, :, int(w * (1 - frac)):] = True
        for i, lf in case["full"]:
            if lf == l:
                m[i] = True
        parts.append(m.flatten(1))
    return torch.cat(parts, 1)


def geometry(case):
    sizes = [h * w for h, w in case["shapes"]]
    starts = [sum(sizes[:l]) for l in range(len(sizes))]
    return starts, sizes


def cell_keys(inds, starts, shapes, strides, cell_px):
    """((cy * cells_x + cx) << 3) | l of each selected token: its spatial cell and level, as the host defines them."""
    st = torch.tensor(starts)
    lvl = torch.bucketize(inds, st, right=True) - 1
    w = torch.tensor([w for _, w in shapes])[lvl]
    s = torch.tensor(strides)[lvl]
    r = inds - st[lvl]
    cells_x = (max(w_ * s_ for (_, w_), s_ in zip(shapes, strides)) + cell_px - 1) // cell_px + 1
    cy, cx = ((r // w) * s + s // 2) // cell_px, ((r % w) * s + s // 2) // cell_px
    return ((cy * cells_x + cx) << 3) | lvl


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- non-GPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["ties", "inf", "flat"])
def test_torch_reference_matches_c_oracle(kind):
    """The torch reference equals the C oracle on finite inputs with many ties, padding, and fills equal to real scores."""
    g = torch.Generator().manual_seed(5)
    for case in (CASES[1], CASES[2], CASES[5]):
        starts, sizes = geometry(case)
        raw = make_scores(kind, case["b"], sizes, g)
        mask = make_mask(case)
        wi, ws, wf = orc.c_salience_select(raw, mask, torch.tensor(starts), torch.tensor(sizes), case["k"])
        ti, ts, tf = torch_salience_select(raw, mask, starts, sizes, case["k"])
        assert torch.equal(ti, wi), (kind, case["id"])
        assert torch.equal(_bits(ts), _bits(ws)) and torch.equal(_bits(tf), _bits(wf)), (kind, case["id"])


def test_case_table_reaches_every_path():
    """Each case takes the path it is named for, and the table reaches all three, with and without a processing order."""
    for c in CASES:
        assert select_path(c["shapes"], c["k"], c["strides"], CELL_PX, c["order"]) == c["path"], c["id"]
    assert {(c["path"], c["order"]) for c in CASES} >= {(1, False), (1, True), (2, True), (3, False), (3, True)}


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pkg():
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


def launched_kernels(fn, expect):
    """Names of the kernels `fn` launches.  The profiler can drop launches near the edges of its window (a window of a
    few short kernels can come back empty), but never records a launch that did not happen.  So each window is padded
    by 20 ms at both ends, `fn` runs twice inside it, and the union over up to five windows is taken, stopping once it
    holds every kernel of `expect`: a path that launches other kernels still shows them, one that misses a kernel of
    `expect` still misses it."""
    from torch.profiler import ProfilerActivity, profile
    got = set()
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.02)
            fn()
            fn()
            torch.cuda.synchronize()
            time.sleep(0.02)
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        got |= {k for k in KERNEL_NAMES if any(k in n for n in names)}  # no kernel name contains another
        if got >= expect:
            break
    return got


def _run(pkg, case, raw, mask):
    starts, sizes = geometry(case)
    widths = [w for _, w in case["shapes"]] if case["order"] else None
    strides = case["strides"] if case["order"] else None
    return pkg.cabi.salience_select(raw, mask, starts, sizes, case["k"], widths, strides, CELL_PX)


_CONFIRMED = {}  # case id -> path seen on the device


def confirm_path(pkg, case):
    """Launch the case once under the profiler: exactly the kernels of its predicted path run."""
    if case["id"] not in _CONFIRMED:
        starts, sizes = geometry(case)
        raw = make_scores("ties", case["b"], sizes, torch.Generator().manual_seed(0)).to(DEV)
        mask = make_mask(case).to(torch.uint8).to(DEV)
        want = expected_kernels(case["path"], case["order"])
        got = launched_kernels(lambda: _run(pkg, case, raw, mask), want)
        assert got == want, (case["id"], got)
        _CONFIRMED[case["id"]] = case["path"]
    return _CONFIRMED[case["id"]]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_salience_select_path(pkg, case):
    """Against the torch reference on every adversarial kind: indices exactly, scores and foreground bit for bit (int32
    views, so -0 and NaN payloads count); the processing order is a permutation along which the cell key never decreases
    (a stable argsort of it on paths 2 and 3); its prefixes equal filtering; a repeated call gives the same bits."""
    assert confirm_path(pkg, case) == case["path"]
    starts, sizes = geometry(case)
    b, K = case["b"], sum(case["k"])
    mask = make_mask(case)
    mask_d = mask.to(torch.uint8).to(DEV)
    g = torch.Generator().manual_seed(1)
    for kind in KINDS:
        raw = make_scores(kind, b, sizes, g)
        raw_d = raw.to(DEV)
        wi, ws, wf = torch_salience_select(raw, mask, starts, sizes, case["k"])
        inds, score, fg, order = _run(pkg, case, raw_d, mask_d)
        assert torch.equal(inds.cpu(), wi), kind
        assert torch.equal(_bits(score.cpu()), _bits(ws)), kind
        assert torch.equal(_bits(fg.cpu()), _bits(wf)), kind
        again = _run(pkg, case, raw_d, mask_d)
        assert torch.equal(again[0], inds) and torch.equal(_bits(again[1]), _bits(score)) and torch.equal(_bits(again[2]), _bits(fg))
        if not case["order"] or K == 0:
            assert order is None
            continue
        oc = order.long().cpu()
        assert torch.equal(oc.sort(1)[0], torch.arange(K).expand(b, K)), kind  # a permutation of range(K)
        key = cell_keys(wi, starts, case["shapes"], case["strides"], CELL_PX)
        along = key.gather(1, oc)
        assert (along[:, 1:] >= along[:, :-1]).all(), kind
        if case["path"] != 1:  # stable sorts; the rank-merge path fills each cell bin in atomic order
            assert torch.equal(oc, torch.sort(key, dim=1, stable=True)[1]), kind
            assert torch.equal(again[3], order), kind
        nqs = [K, 3 * K // 5, K // 5]
        for nq, p in zip(nqs, pkg.cabi.order_prefixes(order, nqs)):
            for i in range(b):
                assert torch.equal(p[i].cpu().long(), oc[i][oc[i] < nq]), (kind, nq)


@pytest.mark.gpu
def test_every_path_reached(pkg):
    """The device took all three paths, with and without a processing order (confirmed by the kernels it launched)."""
    reached = {(confirm_path(pkg, c), c["order"]) for c in CASES}
    assert reached >= {(1, False), (1, True), (2, True), (3, False), (3, True)}, sorted(reached)


@pytest.mark.gpu
@pytest.mark.parametrize("seg,n,k", [(1, 1, 1), (3, 37, 37), (2, 1000, 1000), (2, 22323, 300), (2, 4099, 4096),
                                     (2, 5000, 4097), (1, 5003, 5003), (2, 70001, 8000)])
def test_topk_desc_value_edges(pkg, seg, n, k):
    """Both paths of sdetr_topk_desc (select + bitonic for k <= 4096, LSD sort above) equal a stable descending sort on
    every adversarial kind, NaNs of either sign first."""
    g = torch.Generator().manual_seed(n)
    want_kernel = {"topk_select_kernel"} if k <= 4096 else {"topk_kernel"}
    s = make_scores("ties", seg, [n], g).to(DEV)
    assert launched_kernels(lambda: pkg.cabi.topk_desc(s, k), want_kernel) == want_kernel
    for kind in KINDS:
        s = make_scores(kind, seg, [n], g)
        want = torch.sort(s, dim=1, descending=True, stable=True)[1][:, :k]
        assert torch.equal(pkg.cabi.topk_desc(s.to(DEV), k).cpu(), want), kind


@pytest.mark.gpu
def test_five_scale_1333_module_takes_radix_path(pkg):
    """The tiny-width model at the 5-scale strides (4, 8, 16, 32) on a 1333 x 1333 padded batch: K = 75 753 in 38 slices,
    so the module selects on path 3.  Its selection equals the oracle's on the model's own scores."""
    from salience_detr_b200.salience_transformer import TILE_CELL_PX
    from salience_detr_b200.synthetic import build_model, level_shapes, sine_position_embedding
    model = build_model(embed_dim=64, d_ffn=128, heads=TINY_CFG["heads"], points=TINY_CFG["points"],
                        layers=TINY_CFG["num_layers"], topk_sa=TINY_CFG["topk_sa"],
                        level_filter_ratio=TINY_CFG["level_filter_ratio"], layer_filter_ratio=TINY_CFG["layer_filter_ratio"],
                        max_num_embedding=500, strides=(4, 8, 16, 32)).to(DEV)
    g = torch.Generator().manual_seed(2)
    full = torch.ones(2, 1333, 1333, dtype=torch.bool)
    full[0] = False
    full[1, :800, :1200] = False
    feats, masks, pos = [], [], []
    for h, w in level_shapes(1333, 1333, (4, 8, 16, 32)):
        m = torch.nn.functional.interpolate(full[None].float(), size=(h, w))[0].to(torch.bool)
        feats.append(torch.randn(2, 64, h, w, generator=g).to(DEV))
        masks.append(m.to(DEV))
        pos.append(sine_position_embedding(m, 32).to(DEV))
    with torch.no_grad():
        mem, aux = model.forward_encoder(feats, masks, pos)
    plan = aux["plan"]
    assert plan.num_selected == 75753
    assert select_path(plan.shapes_list, plan.level_token_nums, plan.level_stride, TILE_CELL_PX, True) == 3
    wi, _, wf = orc.c_salience_select(aux["raw_score"].cpu(), plan.mask_flat.cpu(), plan.level_start_index.cpu(),
                                      torch.tensor(plan.level_size), plan.level_token_nums)
    assert torch.equal(aux["selected_inds"].cpu(), wi)
    assert torch.equal(_bits(aux["foreground_score"].cpu()), _bits(wf))
    assert torch.isfinite(mem).all()
