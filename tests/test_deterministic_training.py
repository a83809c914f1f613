"""Bit-reproducible training under ``torch.use_deterministic_algorithms(True)``: the fixed-point MSDA core backward
(``sdetr_msda_backward_deterministic``), the gather-form backward of the salience filter's score upsample
(``sdetr_upsample_bilinear_ac_backward``), and whole training steps that must give the same gradient bits twice.

The module-level training checks run in a subprocess: the deterministic mode and ``CUBLAS_WORKSPACE_CONFIG`` are process-wide
and must be set before the first cuBLAS call."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT, load_golden

DEV = "cuda:0"


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as entry
    entry.build()
    import salience_detr_b200 as p
    p.cabi.lib()
    return p


# ---- no GPU needed: argument checks run on the host before any CUDA call ---------------------------------------------------
def test_argument_validation(pkg):
    lib = pkg.cabi.lib()
    buf = (ctypes.c_float * 1024)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    p16 = (p + 15) // 16 * 16
    ws = lib.sdetr_msda_backward_deterministic_workspace(2, 100, 8, 32)
    assert ws >= 8 * 2 * 100 * 8 * 32
    rc = lib.sdetr_msda_backward_deterministic(None, p16, p16, p16, p16, p16, p16, p16, p16, 2, 100, 8, 32, 4, 10, 4,
                                               p16, ws, None)
    assert rc == -1 and b"null pointer" in lib.sdetr_last_error()
    rc = lib.sdetr_msda_backward_deterministic(*[p16] * 9, 2, 100, 8, 32, 4, 10, 4, p16, ws - 1, None)
    assert rc == -4 and b"workspace" in lib.sdetr_last_error()
    rc = lib.sdetr_msda_backward_deterministic(*[p16] * 9, 2, 100, 8, 24, 4, 10, 4, p16, 1 << 40, None)
    assert rc == -2 and b"head_dim 24" in lib.sdetr_last_error()
    rc = lib.sdetr_msda_backward_deterministic(*[p16] * 9, 2, 100, 8, 32, 4, 10, 4, None, ws, None)
    assert rc == -1
    rc = lib.sdetr_msda_backward_deterministic(*[p16] * 9, 2, 100, 8, 32, 9, 10, 4, p16, ws, None)
    assert rc == -2 and b"levels" in lib.sdetr_last_error()
    rc = lib.sdetr_upsample_bilinear_ac_backward(None, 2, 10, 12, 5, 6, p16, None)
    assert rc == -1 and b"null pointer" in lib.sdetr_last_error()
    rc = lib.sdetr_upsample_bilinear_ac_backward(p16, 2, 10, 0, 5, 6, p16, None)
    assert rc == -1 and b"non-positive" in lib.sdetr_last_error()


def test_workspace_size(pkg):
    lib = pkg.cabi.lib()
    for b, nv, m, d in ((2, 22323, 8, 32), (1, 1, 1, 4), (3, 4080, 2, 128)):
        assert lib.sdetr_msda_backward_deterministic_workspace(b, nv, m, d) >= 8 * b * nv * m * d
    assert lib.sdetr_msda_backward_deterministic_workspace(0, 10, 8, 32) == 0


def test_library_exports_and_stays_sm90a_torch_free(pkg):
    cdll = ctypes.CDLL(pkg.cabi.LIB_PATH)
    for s in ("sdetr_msda_backward_deterministic", "sdetr_msda_backward_deterministic_workspace",
              "sdetr_upsample_bilinear_ac_backward"):
        assert hasattr(cdll, s)
    out = subprocess.run(["cuobjdump", "--list-elf", pkg.cabi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    ldd = subprocess.run(["ldd", pkg.cabi.LIB_PATH], capture_output=True, text=True).stdout
    # the names and paths of the libraries it links, without the load addresses (whose hex digits can spell "c10")
    linked = " ".join(line.split(" (0x")[0] for line in ldd.splitlines())
    assert "torch" not in linked and "c10" not in linked


# ---- MSDA core backward on the H100 ------------------------------------------------------------------------------------------
def _msda_inputs(b, shapes, m, d, nq, p, seed):
    g = torch.Generator().manual_seed(seed)
    st = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([st.new_zeros(1), st.prod(1).cumsum(0)[:-1]])
    nv = int(st.prod(1).sum())
    L = len(shapes)
    value = torch.randn(b, nv, m, d, generator=g)
    loc = torch.rand(b, nq, m, L, p, 2, generator=g) * 1.2 - 0.1
    attn = torch.randn(b, nq, m, L * p, generator=g).softmax(-1).view(b, nq, m, L, p)
    gout = torch.randn(b, nq, m * d, generator=torch.Generator().manual_seed(seed + 1))
    return value, st, lsi, loc, attn, gout


# the shapes of test_gpu_parity.py::test_msda_backward_vs_oracle, plus the degenerate 1x1 maps
CASES = [
    (2, [(16, 20), (8, 10), (4, 5), (2, 3)], 8, 32, 77, 4),
    (1, [(20, 24), (10, 12), (5, 6), (3, 3), (2, 2)], 4, 32, 130, 4),
    (2, [(9, 7), (5, 4), (3, 2), (1, 1)], 2, 64, 33, 4),
    (1, [(7, 5), (4, 3)], 2, 16, 23, 2),
    (1, [(1, 1), (1, 1), (1, 1), (1, 1)], 8, 32, 5, 4),
    (1, [(3, 2)], 1, 4, 3, 1),
    (1, [(4, 3), (2, 2)], 2, 8, 11, 3),
    (1, [(5, 4), (2, 2)], 2, 128, 17, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_deterministic_backward_vs_oracle(pkg, case):
    from oracle import oracle as orc
    b, shapes, m, d, nq, p = case
    value, st, lsi, loc, attn, gout = _msda_inputs(b, shapes, m, d, nq, p, seed=100 + nq)
    wv, wl, wa = orc.c_msda_backward(value, st, lsi, loc, attn, gout)
    args = [t.to(DEV) for t in (value, st, lsi, loc, attn, gout)]
    gv, gl, ga = pkg.cabi.msda_backward_deterministic(*args)
    assert (gv.cpu() - wv).abs().max() < 2e-4 * max(1.0, wv.abs().max().item())
    assert (ga.cpu() - wa).abs().max() < 1e-4
    assert (gl.cpu() - wl).abs().max() / wl.abs().max() < 1e-5
    _, al, aa = pkg.cabi.msda_backward(*args)
    assert torch.equal(gl, al) and torch.equal(ga, aa)  # the same code computes them


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["msda_core_a", "msda_core_b"])
def test_deterministic_backward_vs_reference_golden(pkg, name):
    g, _ = load_golden(name)
    dv = {k: v.to(DEV) for k, v in g.items()}
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        gv, gl, ga = pkg.ms_deform_attn_backward(dv["value"], dv["shapes"], dv["lsi"], dv["loc"], dv["attn"], dv["grad_out"], 64)
    finally:
        torch.use_deterministic_algorithms(False)
    assert (gv.cpu() - g["grad_value"]).abs().max() < 1e-4
    assert (ga.cpu() - g["grad_attn"]).abs().max() < 1e-4
    assert (gl.cpu() - g["grad_loc"]).abs().max() / g["grad_loc"].abs().max() < 1e-5
    _, al, aa = pkg.cabi.msda_backward(dv["value"], dv["shapes"], dv["lsi"], dv["loc"], dv["attn"], dv["grad_out"])
    assert torch.equal(gl, al) and torch.equal(ga, aa)


@pytest.mark.gpu
def test_bits_do_not_depend_on_query_order_or_repetition(pkg):
    """Collision-heavy: 3000 queries x 2 heads x 4 points sample two tiny levels, so every value element receives hundreds to
    thousands of contributions.  Repeated calls and any permutation of the queries give the same grad_value bits."""
    value, st, lsi, loc, attn, gout = [t.to(DEV) for t in _msda_inputs(1, [(2, 3), (1, 1)], 2, 32, 3000, 4, seed=5)]
    loc = (loc * 0.6 + 0.2).contiguous()  # mostly inside the maps
    gv0, gl0, ga0 = pkg.cabi.msda_backward_deterministic(value, st, lsi, loc, attn, gout)
    for _ in range(3):
        gv, gl, ga = pkg.cabi.msda_backward_deterministic(value, st, lsi, loc, attn, gout)
        assert torch.equal(gv, gv0) and torch.equal(gl, gl0) and torch.equal(ga, ga0)
    atomic = [pkg.cabi.msda_backward(value, st, lsi, loc, attn, gout)[0] for _ in range(2)]
    assert (gv0 - atomic[0]).abs().max() < 1e-4 * max(1.0, atomic[0].abs().max().item())
    for seed in range(3):
        perm = torch.randperm(3000, generator=torch.Generator().manual_seed(seed)).to(DEV)
        gv, gl, ga = pkg.cabi.msda_backward_deterministic(value, st, lsi, loc[:, perm].contiguous(), attn[:, perm].contiguous(),
                                                          gout[:, perm].contiguous())
        assert torch.equal(gv, gv0), seed
        assert torch.equal(gl, gl0[:, perm]) and torch.equal(ga, ga0[:, perm])


@pytest.mark.gpu
def test_graph_capture_replays_the_eager_bits(pkg):
    args = [t.to(DEV) for t in _msda_inputs(2, [(16, 20), (8, 10), (4, 5), (2, 3)], 8, 32, 77, 4, seed=3)]
    want = pkg.cabi.msda_backward_deterministic(*args)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        pkg.cabi.msda_backward_deterministic(*args)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = pkg.cabi.msda_backward_deterministic(*args)
    for _ in range(2):
        for t in got:
            t.fill_(7.0)
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, w) for a, w in zip(got, want))


@pytest.mark.gpu
def test_empty_query_set_and_non_finite_inputs(pkg):
    value, st, lsi, loc, attn, gout = [t.to(DEV) for t in _msda_inputs(2, [(16, 20), (8, 10), (4, 5), (2, 3)], 8, 32, 50, 4, seed=3)]
    gv, gl, ga = pkg.cabi.msda_backward_deterministic(value, st, lsi, loc[:, :0].contiguous(), attn[:, :0].contiguous(),
                                                      gout[:, :0].contiguous())
    assert gv.shape == value.shape and bool((gv == 0).all()) and gl.numel() == 0 and ga.numel() == 0
    # non-finite sampling locations contribute exactly 0, as in the atomic kernel
    bad = loc.clone()
    bad[0, 3, 2, 1, 0, 0] = float("nan")
    bad[1, 7, 5, 3, 2, 1] = float("inf")
    bad[1, 9, 0, 0, 1, :] = -float("inf")
    gv, gl, ga = pkg.cabi.msda_backward_deterministic(value, st, lsi, bad, attn, gout)
    far = torch.nan_to_num(bad, nan=-9.0, posinf=9.0, neginf=-9.0)  # out of the maps: contributes nothing
    wv, wl, wa = pkg.cabi.msda_backward_deterministic(value, st, lsi, far, attn, gout)
    assert torch.isfinite(gv).all() and torch.equal(gv, wv)
    av, al, aa = pkg.cabi.msda_backward(value, st, lsi, bad, attn, gout)
    assert torch.equal(gl, al) and torch.equal(ga, aa)
    # a non-finite grad_output or attention weight: every grad_value entry is NaN
    for which in ("gout", "attn"):
        g2, a2 = gout.clone(), attn.clone()
        (g2 if which == "gout" else a2).view(-1)[123] = float("inf") if which == "gout" else float("nan")
        gv, _, _ = pkg.cabi.msda_backward_deterministic(value, st, lsi, loc, a2, g2)
        assert bool(torch.isnan(gv).all()), which


# ---- upsample backward ------------------------------------------------------------------------------------------------------
def _tiny_pairs():
    g, _ = load_golden("encoder_tiny_even")
    hw = [tuple(g[f"feat{i}"].shape[-2:]) for i in range(4)]
    return [(hw[i + 1], hw[i]) for i in range(3)]


UPSAMPLE_PAIRS = ([((50, 84), (100, 168)), ((25, 42), (50, 84)), ((13, 21), (25, 42))] +
                  [((1, 1), (3, 5)), ((7, 9), (7, 9)), ((9, 7), (4, 3)), ((1, 6), (4, 11)), ((5, 1), (5, 1))])


@pytest.mark.gpu
@pytest.mark.parametrize("pair", UPSAMPLE_PAIRS + ["tiny"])
def test_upsample_backward_vs_autograd(pkg, pair):
    pairs = _tiny_pairs() if pair == "tiny" else [pair]
    for (hc, wc), (h, w) in pairs:
        gen = torch.Generator().manual_seed(hc * 100 + w)
        x = torch.randn(2, 1, hc, wc, generator=gen, dtype=torch.float64, requires_grad=True)
        grad = torch.randn(2, 1, h, w, generator=gen)
        torch.nn.functional.interpolate(x, size=(h, w), mode="bilinear", align_corners=True).backward(grad.double())
        got = pkg.cabi.upsample_bilinear_ac_backward(grad.to(DEV), hc, wc)
        assert got.shape == (2, 1, hc, wc)
        assert (got.double().cpu() - x.grad).abs().max() < 1e-5 * max(1.0, x.grad.abs().max().item()), ((hc, wc), (h, w))
        assert torch.equal(pkg.cabi.upsample_bilinear_ac_backward(grad.to(DEV), hc, wc), got)


@pytest.mark.gpu
def test_upsample_function_forward_bits_and_backward(pkg):
    from salience_detr_b200.salience_transformer import UpsampleBilinearAC
    x = torch.randn(2, 1, 13, 21, device=DEV, requires_grad=True)
    y = UpsampleBilinearAC.apply(x, (25, 42))
    assert torch.equal(y, torch.nn.functional.interpolate(x.detach(), size=(25, 42), mode="bilinear", align_corners=True))
    g = torch.randn_like(y)
    y.backward(g)
    assert torch.equal(x.grad, pkg.cabi.upsample_bilinear_ac_backward(g, 13, 21))


# ---- routing ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_flag_selects_the_backward(pkg, monkeypatch):
    """Flag off: the atomic sdetr_msda_backward runs (nothing changes); flag on (either warn_only): the deterministic one."""
    calls = []
    for name in ("msda_backward", "msda_backward_deterministic"):
        fn = getattr(pkg.cabi, name)
        monkeypatch.setattr(pkg.cabi, name, lambda *a, _fn=fn, _n=name: calls.append(_n) or _fn(*a))
    value, st, lsi, loc, attn, _ = _msda_inputs(1, [(6, 5), (3, 3)], 2, 32, 9, 2, seed=3)

    def step():
        v, l, a = (t.to(DEV).requires_grad_(True) for t in (value, loc, attn))
        pkg.MultiScaleDeformableAttnFunction.apply(v, st.to(DEV), lsi.to(DEV), l, a, 64).square().sum().backward()
        return v.grad, l.grad, a.grad

    assert not torch.are_deterministic_algorithms_enabled()
    off = step()
    assert calls == ["msda_backward"]
    for warn_only in (True, False):
        calls.clear()
        torch.use_deterministic_algorithms(True, warn_only=warn_only)
        try:
            on = step()
        finally:
            torch.use_deterministic_algorithms(False)
        assert calls == ["msda_backward_deterministic"]
        assert torch.equal(on[1], off[1]) and torch.equal(on[2], off[2]) and (on[0] - off[0]).abs().max() < 1e-5


# ---- whole training steps, strict deterministic mode, in a subprocess ---------------------------------------------------------
def _digest(t):
    return hashlib.sha1(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def _grads(named_params, extra=()):
    out = {n: p.grad.detach().clone() for n, p in named_params if p.grad is not None}
    for i, t in enumerate(extra):
        if t.grad is not None:
            out[f"input{i}"] = t.grad.detach().clone()
    return out


class _OpLog(torch.utils._python_dispatch.TorchDispatchMode):
    """Digest of every aten op's outputs, in call order (forward and backward): the first op whose bits differ between two
    runs is where the non-determinism enters (ops of the C-ABI library show up as the first torch op reading their output)."""

    def __init__(self):
        super().__init__()
        self.log = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        flat = out if isinstance(out, (tuple, list)) else (out,)
        self.log.append((str(func), tuple(_digest(t) for t in flat if torch.is_tensor(t) and t.is_cuda and t.numel())))
        return out


def _case_tiny(pkg):
    from conftest import load_golden as lg
    g, sd = lg("encoder_tiny_even")
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(64, 128, 0.0, 2, topk_sa=20), 3, 40)
    tr = pkg.SalienceTransformer(enc, num_classes=11, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
                                 layer_filter_ratio=(1.0, 0.6, 0.3)).to(DEV)
    assert not tr.load_state_dict(sd, strict=False).missing_keys
    tr.train()
    feats0 = [g[f"feat{i}"].to(DEV) for i in range(4)]
    masks = [g[f"mask{i}"].to(DEV) for i in range(4)]
    pos = [g[f"pos{i}"].to(DEV) for i in range(4)]

    def step():
        tr.zero_grad(set_to_none=True)
        feats = [f.clone().requires_grad_(True) for f in feats0]
        mem, _ = tr.forward_encoder(feats, masks, pos)
        mem.square().mean().backward()
        return _grads(tr.named_parameters(), feats)

    def check(grads):  # the tolerance of test_gpu_parity.py::test_encoder_training_path_gradients
        gg, _ = lg("encoder_tiny_even_grads")
        n = 0
        for key, want in gg.items():
            if key.startswith("grad."):
                got = grads[key[5:]]
            elif key.startswith("grad_feat"):
                got = grads["input%d" % int(key[9:])]
            else:
                continue
            err = (got.cpu() - want).abs().max().item()
            assert err <= 2e-3 * want.abs().max().item() + 1e-7, (key, err)
            n += 1
        assert n >= 70
    return step, check


def _case_c256(pkg):
    from conftest import C256_CFG, load_c256_golden
    _, sd, (feats, masks, pos) = load_c256_golden()
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(256, 256, 0.0, 8, topk_sa=64), 2, 80)
    tr = pkg.SalienceTransformer(enc, num_classes=11, level_filter_ratio=C256_CFG["level_filter_ratio"],
                                 layer_filter_ratio=C256_CFG["layer_filter_ratio"]).to(DEV)
    tr.load_state_dict(sd, strict=False)
    tr.train()
    feats, masks, pos = [f.to(DEV) for f in feats], [m.to(DEV) for m in masks], [p.to(DEV) for p in pos]
    tc_calls = []
    orig = pkg.cabi.gemm_f16x3_scaled
    pkg.cabi.gemm_f16x3_scaled = lambda *a, **k: tc_calls.append(1) or orig(*a, **k)

    def step():
        tr.zero_grad(set_to_none=True)
        mem, _ = tr.forward_encoder(feats, masks, pos)
        mem.square().mean().backward()
        return _grads(tr.named_parameters())

    def check(grads):
        assert tc_calls, "the C = 256 training step did not take the tensor-core Linear path"
    return step, check


def _case_decoder(pkg):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_decoder_half as tdh
    _, shapes = tdh._golden(False)
    ours = tdh._ours(pkg, shapes).train()
    feats, masks, pos = tdh._inputs(False)

    def step():
        ours.zero_grad(set_to_none=True)
        out = ours(feats, masks, pos, None, None, None)
        loss = sum(t.float().square().mean() for t in list(out[:4]) + list(out[4]) if t.requires_grad)
        loss.backward()
        return _grads(ours.named_parameters())

    return step, lambda grads: None


def _child(case):
    """Runs in the subprocess: two training steps from identical state, strict deterministic mode."""
    torch.use_deterministic_algorithms(True)
    import salience_detr_b200 as pkg
    pkg.cabi.lib()
    calls = {"det": 0, "atomic": 0}
    det, atomic = pkg.cabi.msda_backward_deterministic, pkg.cabi.msda_backward
    pkg.cabi.msda_backward_deterministic = lambda *a: calls.__setitem__("det", calls["det"] + 1) or det(*a)
    pkg.cabi.msda_backward = lambda *a: calls.__setitem__("atomic", calls["atomic"] + 1) or atomic(*a)
    step, check = {"tiny": _case_tiny, "c256": _case_c256, "decoder": _case_decoder}[case](pkg)
    a = step()
    b = step()
    res = {"grads": len(a), "msda_backward_calls": calls, "differ": sorted(k for k in a if not torch.equal(a[k], b.get(k)))}
    res["missing"] = sorted(set(a) ^ set(b))
    if res["differ"]:  # locate the first op whose output bits differ between two runs
        logs = []
        for _ in range(2):
            with _OpLog() as m:
                step()
            logs.append(m.log)
        first = next((i for i, (x, y) in enumerate(zip(*logs)) if x != y), None)
        res["first_differing_op"] = None if first is None else [logs[0][first][0], first, len(logs[0]),
                                                                [op for op, _ in logs[0][max(0, first - 5):first]]]
    check(a)
    print("RESULT " + json.dumps(res))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tiny", "c256", "decoder"])
def test_training_step_is_bit_reproducible(pkg, case):
    """Tiny encoder (gradients also within test_encoder_training_path_gradients' tolerance of the reference's), the real
    width C = 256 (tensor-core Linear path), and the full transformer with the decoder: in strict deterministic mode the step
    raises nothing and two steps from identical state give bit-identical gradients, through the deterministic MSDA backward."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_deterministic_training as t; t._child(%r)"
            % (ROOT, os.path.join(ROOT, "tests"), case))
    r = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    res = json.loads(r.stdout.split("RESULT ", 1)[1].splitlines()[0])
    assert res["grads"] > 0 and not res["missing"], res
    assert not res["differ"], res
    assert res["msda_backward_calls"]["det"] > 0 and res["msda_backward_calls"]["atomic"] == 0, res
