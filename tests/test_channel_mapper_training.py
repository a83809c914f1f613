"""ChannelMapper training in token layout: ChannelMapper.forward_tokens under autograd (channel_mapper._TrainMapper) and its
GroupNorm backward kernel (sdetr_group_norm_tokens_backward).

Gradient tolerances follow tests/test_neck_training.py: each tensor is compared as max|g - g64| / max|g64| against a float64
twin, and the bound is a multiple of the same quantity for the fp32 torch path (forward() on cuDNN with TF32 off)."""
import copy
import ctypes
from collections import OrderedDict

import pytest
import torch
import torch.nn.functional as F

import salience_detr_b200 as pkg
from salience_detr_b200 import backbone as bbm
from salience_detr_b200 import cabi
from salience_detr_b200 import channel_mapper as cmm
from backbone_harness import resnet_backbone, resnet_images
from tools import make_channel_mapper_golden as mcg

DEV = "cuda:0"
FP32_MULTIPLE = 16.0
# the GroupNorm backward kernel against torch's own fp32 CUDA GroupNorm backward, both measured against float64
GN_TORCH_MULTIPLE = 4.0
GN_MAPS = [(1, 1), (3, 5), (1, 7), (12, 20), (100, 168)]
R50 = (512, 1024, 2048)
SMALL_SHAPES = [(10, 14), (5, 7), (3, 4)]
CONFIG2_SHAPES = [(100, 168), (50, 84), (25, 42)]


def _rel(a, ref):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    return float((a - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


# ---- no GPU needed --------------------------------------------------------------------------------------------------------
def test_group_norm_backward_rejects_bad_arguments():
    import __graft_entry__ as entry
    entry.build()
    lib = cabi.lib()
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.cast(buf, ctypes.c_void_p).value + 15) // 16 * 16
    sizes = cabi._host_i32([4, 6])
    ws = lib.sdetr_group_norm_tokens_backward_workspace_floats(2, 256, 32, 2, sizes)
    assert ws == lib.sdetr_group_norm_tokens_workspace_floats(2, 256, 32, 2, sizes) + 2 * 2 * 2 * 32
    good = [p, p, p, 10 * 256, 2, 256, 2, sizes, p, 32, 1e-5, p, p, p, ws, None]

    def call(**kw):
        args = list(good)
        for i, v in kw.items():
            args[int(i[1:])] = v
        return lib.sdetr_group_norm_tokens_backward(*args)

    for i in (0, 1, 2, 7, 8, 13):
        assert call(**{f"a{i}": None}) == -1 and b"null pointer" in lib.sdetr_last_error()
    assert call(a5=250, a9=25) != 0 and b"multiple of 4" in lib.sdetr_last_error()
    assert call(a5=8192, a9=32) != 0 and b"at most 4096" in lib.sdetr_last_error()
    assert call(a9=24) != 0 and b"divisible" in lib.sdetr_last_error()
    assert call(a7=cabi._host_i32([4, 0])) != 0 and b"empty level" in lib.sdetr_last_error()
    assert call(a2=p + 4) != 0 and b"16-byte aligned" in lib.sdetr_last_error()
    assert call(a3=10 * 256 + 2) != 0 and b"16-byte aligned" in lib.sdetr_last_error()
    assert call(a3=9 * 256) != 0 and b"pitch below" in lib.sdetr_last_error()
    assert call(a14=ws - 1) != 0 and b"workspace too small" in lib.sdetr_last_error()


def test_training_tokens_supported_rejects_cpu_and_float64():
    m = mcg.build(pkg.ChannelMapper).train()
    for inputs in (mcg.inputs(), OrderedDict((k, v.double()) for k, v in mcg.inputs().items())):
        assert not m.training_tokens_supported(inputs)
        with pytest.raises(RuntimeError, match="needs forward"):
            m.forward_tokens(inputs)


# ---- GPU: the GroupNorm backward kernel -----------------------------------------------------------------------------------
def _gn_case(c, groups, b, seed):
    """a (b, lead + Nv, C) buffer with GN_MAPS levels after `lead` rows, level 3 at 1e4 + N(0, 1); dy, gamma"""
    gen = torch.Generator().manual_seed(seed)
    sizes = [h * w for h, w in GN_MAPS]
    lead = 7
    x = torch.randn(b, lead + sum(sizes), c, generator=gen)
    s3 = lead + sum(sizes[:3])
    x[:, s3:s3 + sizes[3]] += 1e4
    x[:, lead + sum(sizes[:4]):] *= 3.0
    dy = torch.randn(b, lead + sum(sizes), c, generator=gen)
    gamma = 1.0 + 0.3 * torch.randn(len(sizes), c, generator=gen)
    return x, dy, gamma, sizes, lead


def _gn_autograd(x, dy, gamma, sizes, groups, eps, dtype, device):
    """(dx, dgamma, dbeta) of F.group_norm per level in ``dtype`` on ``device``; x, dy: (b, Nv, C) token rows"""
    dxs, dgs, dbs, s = [], [], [], 0
    for l, n in enumerate(sizes):
        xl = x[:, s:s + n].to(device, dtype).transpose(1, 2).contiguous().requires_grad_(True)
        g = gamma[l].to(device, dtype).requires_grad_(True)
        bt = torch.zeros_like(g).requires_grad_(True)
        y = F.group_norm(xl, groups, g, bt, eps)
        dx, dg, db = torch.autograd.grad(y, (xl, g, bt), dy[:, s:s + n].to(device, dtype).transpose(1, 2))
        dxs.append(dx.transpose(1, 2))
        dgs.append(dg)
        dbs.append(db)
        s += n
    return torch.cat(dxs, 1), torch.stack(dgs), torch.stack(dbs)


@pytest.mark.gpu
@pytest.mark.parametrize("c,groups", [(256, 32), (256, 16), (512, 32), (512, 16), (192, 32), (192, 16)])
@pytest.mark.parametrize("b", [1, 2])
def test_group_norm_backward_vs_fp64(c, groups, b):
    """dx, dgamma, dbeta on a token-range view of a larger buffer (the leading rows stay untouched): within GN_TORCH_MULTIPLE
    of torch's fp32 CUDA GroupNorm backward's error against float64 autograd, each as a max relative error; bit-identical on a
    second run"""
    eps = 1e-5
    x, dy, gamma, sizes, lead = _gn_case(c, groups, b, c + groups + b)
    want = _gn_autograd(x[:, lead:], dy[:, lead:], gamma, sizes, groups, eps, torch.float64, "cpu")
    t32 = _gn_autograd(x[:, lead:], dy[:, lead:], gamma, sizes, groups, eps, torch.float32, DEV)
    xd, dyd, gd = x.to(DEV), dy.to(DEV), gamma.to(DEV)
    dxbuf = torch.full_like(xd, float("nan"))
    got = cabi.group_norm_tokens_backward(dyd[:, lead:], xd[:, lead:], sizes, gd, groups, eps, dx=dxbuf[:, lead:])
    assert got[0].data_ptr() == dxbuf.data_ptr() + lead * c * 4
    assert bool(dxbuf[:, :lead].isnan().all())
    ratios = []
    for name, a, a32, a64 in zip(("dx", "dgamma", "dbeta"), got, t32, want):
        e, e32 = _rel(a, a64), _rel(a32, a64)
        ratios.append(e / max(e32, 1e-12))
        assert e <= GN_TORCH_MULTIPLE * e32 + 2.0 ** -22, (name, e, e32)
    print(f"group_norm_tokens_backward C={c} G={groups} b={b}: error / torch fp32's (dx, dgamma, dbeta) = "
          + ", ".join(f"{r:.2f}" for r in ratios))
    again = cabi.group_norm_tokens_backward(dyd[:, lead:], xd[:, lead:], sizes, gd, groups, eps,
                                            dx=torch.empty_like(dxbuf)[:, lead:])
    for a, b2 in zip(got, again):
        assert torch.equal(a, b2)


@pytest.mark.gpu
def test_group_norm_backward_aliasing_and_optional_outputs():
    """dx over x or over dy gives the separate dx's bits; dgamma / dbeta may each be skipped without changing the rest"""
    x, dy, gamma, sizes, lead = _gn_case(256, 32, 2, 11)
    x, dy = x[:, lead:].contiguous(), dy[:, lead:].contiguous()
    xd, dyd, gd = x.to(DEV), dy.to(DEV), gamma.to(DEV)
    dx, dg, db = cabi.group_norm_tokens_backward(dyd, xd, sizes, gd, 32, 1e-5)
    xa = xd.clone()
    out = cabi.group_norm_tokens_backward(dyd, xa, sizes, gd, 32, 1e-5, dx=xa)
    assert out[0].data_ptr() == xa.data_ptr() and torch.equal(xa, dx) and torch.equal(out[1], dg) and torch.equal(out[2], db)
    dya = dyd.clone()
    out = cabi.group_norm_tokens_backward(dya, xd, sizes, gd, 32, 1e-5, dx=dya)
    assert torch.equal(dya, dx) and torch.equal(out[1], dg) and torch.equal(out[2], db)
    for want_g, want_b in ((True, False), (False, True), (False, False)):
        n0 = cabi.launch_count()
        d, g, bb = cabi.group_norm_tokens_backward(dyd, xd, sizes, gd, 32, 1e-5, dgamma=want_g, dbeta=want_b)
        assert cabi.launch_count() - n0 == 5 + (want_g or want_b)
        assert torch.equal(d, dx) and (g is None) != want_g and (bb is None) != want_b
        assert g is None or torch.equal(g, dg)
        assert bb is None or torch.equal(bb, db)


@pytest.mark.gpu
def test_group_norm_backward_nan_placement_matches_torch():
    """a NaN in x poisons its (image, level, group) of dx and that group's channels of dgamma; a NaN in dy poisons its
    (image, level, group) of dx and its channel of dgamma and dbeta -- torch's placement"""
    c, groups = 256, 32
    x, dy, gamma, sizes, lead = _gn_case(c, groups, 2, 5)
    x, dy = x[:, lead:].contiguous(), dy[:, lead:].contiguous()
    x[0, sizes[0] + 3, 17] = float("nan")   # image 0, level 1, group 2
    dy[1, sum(sizes[:4]) + 100, 200] = float("nan")  # image 1, level 4, group 25
    want = _gn_autograd(x, dy, gamma, sizes, groups, 1e-5, torch.float32, DEV)
    got = cabi.group_norm_tokens_backward(dy.to(DEV), x.to(DEV), sizes, gamma.to(DEV), groups, 1e-5)
    for a, w in zip(got, want):
        assert torch.equal(a.isnan(), w.isnan())
        assert 0 < int(a.isnan().sum()) < a.numel()


# ---- GPU: the module ------------------------------------------------------------------------------------------------------
def _mapper(cin=R50, num_outs=None, **kw):
    torch.manual_seed(5)
    return mcg.perturb_affine(pkg.ChannelMapper(list(cin), 256, num_outs or len(cin) + 1, **kw)).to(DEV).train()


def _inputs(cin, shapes, channels_last, requires_grad, b=2, seed=3):
    g = torch.Generator().manual_seed(seed)
    fmt = torch.channels_last if channels_last else torch.contiguous_format
    return OrderedDict((str(i), torch.randn(b, c, h, w, generator=g).to(DEV).contiguous(memory_format=fmt).requires_grad_(requires_grad))
                       for i, (c, (h, w)) in enumerate(zip(cin, shapes)))


def _tokens(outs):
    return torch.cat([o.flatten(2).transpose(1, 2) for o in outs], 1)


def _step(m, inputs, R, tokens):
    """forward + backward of sum(out * R) -> (out tokens, [input gradients] + every parameter's gradient)"""
    xs = [x for x in inputs.values() if x.requires_grad]
    out = m.forward_tokens(inputs)[0] if tokens else _tokens(m(inputs))
    grads = torch.autograd.grad((out * R.to(out.dtype)).sum(), xs + list(m.parameters()))
    return out.detach(), list(grads)


class _NoTF32:
    def __enter__(self):
        self.prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32 = self.prev


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last", [False, True])
def test_training_output_bit_identical_to_inference(channels_last):
    m = _mapper()
    inputs = _inputs(R50, SMALL_SHAPES, channels_last, True)
    with torch.no_grad():
        want, shapes = m.forward_tokens(inputs)
    assert m.training_tokens_supported(inputs) and not m.tokens_supported(inputs)
    got, shapes2 = m.forward_tokens(inputs)
    assert got.requires_grad and shapes2 == shapes and torch.equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("shapes", ["small", "config2"])
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("input_grad", [False, True])
def test_training_gradients_vs_fp64(shapes, channels_last, input_grad):
    """output, input gradients, every convolution weight gradient and the GroupNorm weight and bias gradients: within
    FP32_MULTIPLE of forward()'s error on cuDNN fp32 (TF32 off), both against forward() in float64; input gradients come back
    in the input's layout"""
    shp = SMALL_SHAPES if shapes == "small" else CONFIG2_SHAPES
    m = _mapper()
    inputs = _inputs(R50, shp, channels_last, input_grad)
    nv = sum(h * w for h, w in shp) + sum(((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) for h, w in shp[-1:])
    R = torch.randn(2, nv, 256, generator=torch.Generator().manual_seed(8)).to(DEV)
    m32, m64 = copy.deepcopy(m), copy.deepcopy(m).double()
    in64 = OrderedDict((k, v.detach().double().requires_grad_(input_grad)) for k, v in inputs.items())
    with _NoTF32():
        out, gr = _step(m, inputs, R, True)
        o32, g32 = _step(m32, inputs, R, False)
        o64, g64 = _step(m64, in64, R.double(), False)
    names = [f"grad input {k}" for k, v in inputs.items() if v.requires_grad] + [n for n, _ in m.named_parameters()]
    worst = 0.0
    for name, a, a32, a64 in zip(["out"] + names, [out] + gr, [o32] + g32, [o64] + g64):
        e, e32 = _rel(a, a64), _rel(a32, a64)
        worst = max(worst, e / (e32 + 1e-7))
        assert e <= FP32_MULTIPLE * e32 + 1e-7, (name, e, e32)
    for x, g in zip((v for v in inputs.values() if v.requires_grad), gr):
        assert g.shape == x.shape and g.is_contiguous(memory_format=torch.channels_last if channels_last else torch.contiguous_format)
    print(f"{shapes} channels_last={channels_last} input_grad={input_grad}: worst error / fp32 error = {worst:.2f}")


FROZEN = {
    "conv1": ["convs.1.0.weight"],
    "gn_weight2_bias0": ["convs.2.1.weight", "convs.0.1.bias"],
    "all_gn": [f"convs.{i}.1.{p}" for i in range(4) for p in ("weight", "bias")],
    "extra_conv_and_gn": ["convs.3.0.weight", "convs.3.1.weight", "convs.3.1.bias"],
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(FROZEN))
def test_frozen_parameters_get_no_gradient(case):
    """frozen parameters keep .grad None; the others get the unfrozen run's bits; launches as launches_per_training_step"""
    m = _mapper()
    inputs = _inputs(R50, SMALL_SHAPES, True, True)
    R = torch.randn(2, 140 + 35 + 12 + 4, 256, generator=torch.Generator().manual_seed(9)).to(DEV)
    (m.forward_tokens(inputs)[0] * R).sum().backward()
    want = {n: p.grad.clone() for n, p in m.named_parameters()}
    want_x = [x.grad.clone() for x in inputs.values()]
    m.zero_grad(set_to_none=True)
    for x in inputs.values():
        x.grad = None
    params = dict(m.named_parameters())
    for n in FROZEN[case]:
        params[n].requires_grad_(False)
    n0 = cabi.launch_count()
    (m.forward_tokens(inputs)[0] * R).sum().backward()
    assert cabi.launch_count() - n0 == m.launches_per_training_step(inputs)
    for n, p in m.named_parameters():
        assert (p.grad is None) == (n in FROZEN[case]), n
        assert p.grad is None or torch.equal(p.grad, want[n]), n
    for x, w in zip(inputs.values(), want_x):
        assert torch.equal(x.grad, w)


@pytest.mark.gpu
@pytest.mark.parametrize("channels_last,input_grad,num_outs", [(True, True, 4), (False, True, 4), (False, False, 4),
                                                               (True, True, 3), (True, False, 3)])
def test_launch_count_and_no_host_sync(channels_last, input_grad, num_outs):
    m = _mapper(num_outs=num_outs)
    inputs = _inputs(R50, SMALL_SHAPES, channels_last, input_grad)
    out, _ = m.forward_tokens(inputs)
    R = torch.randn(out.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    targets = [x for x in inputs.values() if x.requires_grad] + list(m.parameters())
    want = torch.autograd.grad((out * R).sum(), targets)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = cabi.launch_count()
        out2, _ = m.forward_tokens(inputs)
        got = torch.autograd.grad((out2 * R).sum(), targets)
        n = cabi.launch_count() - n0
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert n == m.launches_per_training_step(inputs)
    assert torch.equal(out, out2) and all(torch.equal(a, b) for a, b in zip(got, want))
    print(f"channels_last={channels_last} input_grad={input_grad} num_outs={num_outs}: {n} library launches per step")


@pytest.mark.gpu
def test_cuda_graph_step_with_sgd_equals_eager():
    """forward + backward + an SGD step in one CUDA graph: the first replay gives the eager step's bits, the second the eager
    step at the updated weights (the weights are split in every call, so the replay sees the update); two eager backwards
    give equal bits, also under torch.use_deterministic_algorithms(True)"""
    m_graph = _mapper()
    m_eager = copy.deepcopy(m_graph)
    inputs = _inputs(R50, SMALL_SHAPES, True, True)
    R = torch.randn(2, 191, 256, generator=torch.Generator().manual_seed(6)).to(DEV)
    xs = list(inputs.values())

    def grads(m):  # the output detached: no autograd graph (nor the inputs' gradient nodes) outlives the step
        out, _ = m.forward_tokens(inputs)
        return [out.detach()] + list(torch.autograd.grad((out * R).sum(), xs + list(m.parameters())))

    g0 = grads(m_eager)
    again = grads(m_eager)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        det = grads(m_eager)
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b, d in zip(g0, again, det):
        assert torch.equal(a, b) and torch.equal(a, d)
    lr = 1e-3 * max(float(p.abs().max()) for p in m_eager.parameters()) / max(float(g.abs().max()) for g in g0[len(xs) + 1:])

    def step(m):
        r = grads(m)
        with torch.no_grad():
            for p, g in zip(m.parameters(), r[len(xs) + 1:]):
                p.sub_(lr * g)
        return r

    w0 = [p.detach().clone() for p in m_graph.parameters()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(m_graph)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    with torch.no_grad():
        for p, w in zip(m_graph.parameters(), w0):
            p.copy_(w)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        static = step(m_graph)
    for it in range(2):
        graph.replay()
        eager = step(m_eager)
        torch.cuda.synchronize()
        for a, b in zip(static, eager):
            assert torch.equal(a, b), it
        for a, b in zip(m_graph.parameters(), m_eager.parameters()):
            assert torch.equal(a, b), it


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["conv_bias", "two_extra_levels", "cpu_inputs", "float64"])
def test_unsupported_training_raises(case):
    m = _mapper(num_outs=5 if case == "two_extra_levels" else None)
    inputs = _inputs(R50, SMALL_SHAPES, True, True)
    if case == "conv_bias":  # set after construction: the reference's init_weights tests `if layer.bias:`
        m.convs[1][0].bias = torch.nn.Parameter(torch.zeros(256, device=DEV))
    elif case == "cpu_inputs":
        inputs = OrderedDict((k, v.detach().cpu().requires_grad_(True)) for k, v in inputs.items())
    elif case == "float64":
        m = m.double()
        inputs = OrderedDict((k, v.detach().double().requires_grad_(True)) for k, v in inputs.items())
    assert not m.training_tokens_supported(inputs)
    with pytest.raises(RuntimeError, match="needs forward"):
        m.forward_tokens(inputs)
    with torch.no_grad():  # the inference predicate is unchanged
        assert m.tokens_supported(inputs) == (case in ("conv_bias", "two_extra_levels"))


@pytest.mark.gpu
def test_backbone_to_mapper_chain():
    """ResNet-50 forward_tokens (training, freeze_indices=(0,)) -> ChannelMapper forward_tokens (training) -> loss: the
    backbone's weight gradients within 16x of cuDNN fp32's error, each against its float64 stand-in (as
    test_backbone_training.py's chain test: the token chain against the same chain with float64 convolution gradients, the
    all-torch chain in fp32 against float64); the mapper's input gradients reach the backbone's backward without a copy"""
    from test_backbone_training import _ExactBackward
    bb = resnet_backbone().to(DEV)
    mapper = _mapper()
    x = resnet_images(2, 97, 131, torch.Generator().manual_seed(12)).to(DEV)

    def trainable(b):
        return [p for p in b.parameters() if p.requires_grad]

    def run(b, mp, xx, tokens):
        if tokens:
            out = mp.forward_tokens(b.forward_tokens(xx))[0]
        else:
            out = _tokens(mp(b(xx)))
        R = torch.randn(out.shape, generator=torch.Generator().manual_seed(13), dtype=torch.float64).to(DEV, out.dtype)
        return torch.autograd.grad((out * R).sum(), trainable(b))

    sent, received = [], []
    orig_m, orig_b = cmm._TrainMapper.backward, bbm._TrainBlocks.backward

    def m_backward(ctx, gY):
        r = orig_m(ctx, gY)
        sent.extend(g.data_ptr() for g in r[1:1 + ctx.run.n_in])
        return r

    def b_backward(ctx, *g):
        received.extend(t.data_ptr() for t in g)
        return orig_b(ctx, *g)

    cmm._TrainMapper.backward, bbm._TrainBlocks.backward = staticmethod(m_backward), staticmethod(b_backward)
    try:
        got = run(bb, mapper, x, True)
    finally:
        cmm._TrainMapper.backward, bbm._TrainBlocks.backward = staticmethod(orig_m), staticmethod(orig_b)
    assert len(sent) == 3 and sorted(sent) == sorted(received)
    with _ExactBackward():
        exact = run(bb, mapper, x, True)
    ref = run(copy.deepcopy(bb).double(), copy.deepcopy(mapper).double(), x.double(), False)
    with _NoTF32():
        fp32 = run(copy.deepcopy(bb), copy.deepcopy(mapper), x, False)
    worst = 0.0
    for (n, _), g, ex, r, a in zip([(n, p) for n, p in bb.named_parameters() if p.requires_grad], got, exact, ref, fp32):
        assert _rel(g, ex) <= 16 * _rel(a, r), (n, _rel(g, ex), _rel(a, r))
        worst = max(worst, _rel(g, ex) / _rel(a, r))
    print(f"backbone -> mapper chain: worst backbone gradient error / cuDNN fp32's = {worst:.2f}")
