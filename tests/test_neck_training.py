"""RepVGG-PluX neck training in token layout: RepVGGPluXNetwork.forward_tokens under autograd and its kernels
(sdetr_conv2d_f16x3_wgrad, sdetr_conv2d_f16x3_dgrad, sdetr_upsample_nearest_concat_backward).

Gradient tolerances follow tests/test_training_gradients.py: each tensor is compared as max|g - g64| / max|g64| against a float64
twin, and the bound is a multiple of the same quantity for the fp32 torch path (forward() on cuDNN with TF32 off)."""
import copy
import ctypes
import json
import os
import subprocess
import sys
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import salience_detr_b200 as pkg
from conftest import GOLDEN, ROOT
from tools import make_neck_golden as mng

DEV = "cuda:0"
C, G = mng.CHANNELS, mng.GROUPS
CONFIG2_SHAPES = [(100, 168), (50, 84), (25, 42), (13, 21)]
# bound on the token path's relative error of every output, gradient and running statistic: this multiple of the fp32
# forward() path's (cuDNN, TF32 off), plus 1e-7.  The 3xFP16 products keep ~22 significand bits against fp32's 24; the largest
# ratio measured on an H100 was 7.4 (eval mode with gradients, a context-gate FC weight).
FP32_MULTIPLE = 16.0


# ---- no GPU needed --------------------------------------------------------------------------------------------------------
def test_training_entry_points_reject_bad_arguments():
    import __graft_entry__ as entry
    entry.build()
    lib = pkg.cabi.lib()
    buf = (ctypes.c_float * 4096)()
    p = (ctypes.cast(buf, ctypes.c_void_p).value + 15) // 16 * 16
    ws = lib.sdetr_conv2d_f16x3_wgrad_workspace_floats(2, 13, 21, 256, 256, 4, 3)
    assert ws >= 256 * 64 * 9
    assert lib.sdetr_conv2d_f16x3_wgrad_workspace_floats(2, 13, 21, 96, 96, 1, 3) == 0
    assert lib.sdetr_conv2d_f16x3_wgrad_workspace_floats(2, 13, 21, 256, 128, 4, 3) == 0  # Cout / groups = 32: rejected below too
    rc = lib.sdetr_conv2d_f16x3_wgrad(p, 1092 * 128, 128, p, p, 4 * 273 * 256, 256, p, 2, 26, 42, 256, 128, 4, 3, 2, None, p,
                                      1 << 30, p, None)
    assert rc != 0 and b"multiples of 64" in lib.sdetr_last_error()
    split = [p, 256, 256, 4, 3, p, p, p, p, p, None]
    for i in (0, 5, 6, 7):
        args = list(split)
        args[i] = None
        assert lib.sdetr_conv2d_f16x3_split_weight(*args) == -1 and b"null pointer" in lib.sdetr_last_error()
    args = list(split)
    args[8] = None  # dgrad_hi without dgrad_lo
    assert lib.sdetr_conv2d_f16x3_split_weight(*args) == -1 and b"go together" in lib.sdetr_last_error()
    args = list(split)
    args[2] = 254
    assert lib.sdetr_conv2d_f16x3_split_weight(*args) == -1 and b"bad sizes" in lib.sdetr_last_error()
    wgrad = lambda *a: lib.sdetr_conv2d_f16x3_wgrad(*a)  # noqa: E731
    good = [p, 1092 * 256, 256, p, p, 4 * 273 * 256, 256, p, 2, 26, 42, 256, 256, 4, 3, 2, None, p, ws, p, None]
    for i, bad in ((0, None), (3, None), (4, None), (17, None), (19, None)):
        args = list(good)
        args[i] = bad
        assert wgrad(*args) == -1 and b"null pointer" in lib.sdetr_last_error()
    args = list(good)
    args[11], args[12] = 96, 96  # Cin / groups = 24
    assert wgrad(*args) != 0 and b"multiples of 64" in lib.sdetr_last_error()
    args = list(good)
    args[2] = 258  # row stride not 16-byte aligned
    assert wgrad(*args) == -1 and b"16-byte aligned" in lib.sdetr_last_error()
    args = list(good)
    args[1] = 6  # image pitch not 16-byte aligned
    assert wgrad(*args) == -1 and b"16-byte aligned" in lib.sdetr_last_error()
    args = list(good)
    args[18] = ws - 1
    assert wgrad(*args) == -1 and b"workspace too small" in lib.sdetr_last_error()
    args = list(good)
    args[15] = 3
    assert wgrad(*args) != 0 and b"stride 1 or 2" in lib.sdetr_last_error()

    # the input gradient of a stride-2 convolution
    dg = [p, 256 * 256, 256, 2, 13, 21, 256, p, p, p, p, None, 0, 0, None, 0, 0, 256, 4, 3, 2, 26, 42, p, 1092 * 256, 256, None]
    for i in (0, 7, 8, 23):
        args = list(dg)
        args[i] = None
        assert lib.sdetr_conv2d_f16x3_dgrad(*args) == -1 and b"null pointer" in lib.sdetr_last_error()
    args = list(dg)
    args[6], args[17] = 160, 160
    assert lib.sdetr_conv2d_f16x3_dgrad(*args) != 0 and b"multiples of 64" in lib.sdetr_last_error()
    args = list(dg)
    args[4] = 12  # dY is not the stride-2 output size of 26 x 42
    assert lib.sdetr_conv2d_f16x3_dgrad(*args) == -1 and b"stride-2 convolution" in lib.sdetr_last_error()
    args = list(dg)
    args[2] = 250
    assert lib.sdetr_conv2d_f16x3_dgrad(*args) == -1 and b"16-byte aligned" in lib.sdetr_last_error()

    up = [p, 1092 * 512, 512, 26, 42, 13, 21, 2, 256, p, 273 * 256, 256, None]
    args = list(up)
    args[0] = None
    assert lib.sdetr_upsample_nearest_concat_backward(*args) == -1 and b"null pointer" in lib.sdetr_last_error()
    args = list(up)
    args[8] = 6
    assert lib.sdetr_upsample_nearest_concat_backward(*args) == -1 and b"bad sizes" in lib.sdetr_last_error()
    args = list(up)
    args[2] = 510
    assert lib.sdetr_upsample_nearest_concat_backward(*args) == -1 and b"16-byte aligned" in lib.sdetr_last_error()


def dgrad_weight(w, groups):
    """(Cout, Cin / groups, k, k) weight -> the (Cin, k, k, Cout / groups) weight whose stride-1 convolution of dY is the input
    gradient: flipped in both spatial axes and transposed per group -- the layout sdetr_conv2d_f16x3_split_weight writes"""
    cout, cin_g, k, _ = w.shape
    return w.reshape(groups, cout // groups, cin_g, k, k).flip(3, 4).permute(0, 2, 3, 4, 1).reshape(groups * cin_g, k, k,
                                                                                                   cout // groups)


@pytest.mark.parametrize("groups", [1, 4])
@pytest.mark.parametrize("k", [1, 3])
def test_dgrad_weight_reproduces_autograd_fp64(groups, k):
    gen = torch.Generator().manual_seed(10 * groups + k)
    cin, cout = 8 * groups, 12 * groups
    x = torch.randn(2, cin, 7, 9, dtype=torch.float64, generator=gen, requires_grad=True)
    w = torch.randn(cout, cin // groups, k, k, dtype=torch.float64, generator=gen)
    gy = torch.randn(2, cout, 7, 9, dtype=torch.float64, generator=gen)
    (want,) = torch.autograd.grad(F.conv2d(x, w, None, 1, k // 2, groups=groups), x, gy)
    wt = dgrad_weight(w, groups)
    assert tuple(wt.shape) == (cin, k, k, cout // groups)
    got = F.conv2d(gy, wt.permute(0, 3, 1, 2), None, 1, k // 2, groups=groups)
    assert (got - want).abs().max() < 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("src,dst", [((13, 21), (25, 42)), ((25, 42), (50, 84)), ((8, 10), (15, 20)), ((7, 11), (20, 30))])
def test_nearest_ranges_match_interpolate_autograd(src, dst):
    x = torch.zeros(1, 1, *src, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(1, 1, *dst, dtype=torch.float64, generator=torch.Generator().manual_seed(src[0]))
    (want,) = torch.autograd.grad(F.interpolate(x, size=dst, mode="nearest"), x, gy)
    (y0, y1), (x0, x1) = pkg.neck.nearest_ranges(src[0], dst[0]), pkg.neck.nearest_ranges(src[1], dst[1])
    got = torch.zeros(src, dtype=torch.float64)
    for sy in range(src[0]):
        for sx in range(src[1]):
            got[sy, sx] = gy[0, 0, y0[sy]:y1[sy], x0[sx]:x1[sx]].sum()
    assert torch.equal(y1[:-1], y0[1:]) and int(y0[0]) == 0 and int(y1[-1]) == dst[0]
    assert (got - want[0, 0]).abs().max() < 1e-12


# ---- GPU: operators -------------------------------------------------------------------------------------------------------
def _slice(t, lvl_rows, n, c0, c):
    """rows [lvl_rows, lvl_rows + n), channels [c0, c0 + c) of a (b, rows, width) tensor: a level slice / channel half"""
    return t[:, lvl_rows:lvl_rows + n, c0:c0 + c]


# (k, stride, groups, Cin, Cout)
OP_KINDS = {"3x3_s1_g4": (3, 1, 4, 256, 256), "3x3_s2_g1": (3, 2, 1, 256, 256), "1x1_s1_g1_2C_C": (1, 1, 1, 512, 256),
            "1x1_s1_g1_64": (1, 1, 1, 64, 64), "3x3_s2_g4_512": (3, 2, 4, 256, 512), "1x1_s2_g4": (1, 2, 4, 256, 256),
            "3x3_s1_g1_128_64": (3, 1, 1, 128, 64)}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(OP_KINDS))
@pytest.mark.parametrize("b", [1, 2])
def test_conv_dgrad_and_wgrad_vs_fp64(kind, b):
    """weight and input gradients of the token convolution against fp64 autograd of F.conv2d.  Operands are a level slice and
    a channel half of wider buffers.  Elementwise bound as test_neck.py::test_conv_kernel_vs_fp64 states it: 2^-17 x the sum of
    the absolute products (the 3xFP16 products keep ~22 bits, k-block sums are added in fp32)."""
    k, stride, groups, cin, cout = OP_KINDS[kind]
    gen = torch.Generator().manual_seed(sum(map(ord, kind)) + b)
    w = (torch.randn(cout, cin // groups, k, k, generator=gen) / (cin // groups * k * k) ** 0.5).to(DEV)
    for h, wd in [(13, 21), (7, 11), (1, 9), (5, 6), (100, 168)]:
        if (h, wd) == (100, 168) and kind not in ("3x3_s1_g4", "3x3_s2_g1"):
            continue
        ho, wo = (h + 2 * (k // 2) - k) // stride + 1, (wd + 2 * (k // 2) - k) // stride + 1
        xbuf = torch.randn(b, h * wd + 11, 2 * cin, generator=gen).to(DEV)
        x = _slice(xbuf, 11, h * wd, cin, cin)  # level slice and channel half
        gbuf = torch.randn(b, ho * wo + 5, cout, generator=gen).to(DEV)
        gy = gbuf[:, 5:]  # level slice
        x64 = x.double().transpose(1, 2).reshape(b, cin, h, wd).requires_grad_(True)
        w64 = w.double().requires_grad_(True)
        g64 = gy.double().transpose(1, 2).reshape(b, cout, ho, wo)
        dx64, dw64 = torch.autograd.grad(F.conv2d(x64, w64, None, stride, k // 2, groups=groups), (x64, w64), g64)
        xa, wa = x64.detach().abs().requires_grad_(True), w64.detach().abs().requires_grad_(True)
        # sums of the absolute products: the gradients of sum(|g| conv(|x|, |w|))
        bdx, bdw = torch.autograd.grad(F.conv2d(xa, wa, None, stride, k // 2, groups=groups), (xa, wa), g64.abs())
        xs = x.detach()
        dw = pkg.cabi.conv2d_f16x3_wgrad(gy, pkg.cabi.pow2_scale(gbuf, 12), xs, pkg.cabi.pow2_scale(xbuf, 12), (h, wd), w.shape,
                                         stride)
        dw2 = pkg.cabi.conv2d_f16x3_wgrad(gy, pkg.cabi.pow2_scale(gbuf, 12), xs, pkg.cabi.pow2_scale(xbuf, 12), (h, wd), w.shape,
                                          stride)
        assert torch.equal(dw, dw2), (kind, h, wd)  # bit-reproducible
        err = (dw.double() - dw64).abs()
        assert bool((err <= 2.0 ** -17 * bdw + 1e-30).all()), (kind, b, h, wd, float(err.max()), float(bdw.max()))
        f_hi, f_lo, w_hi, w_lo, w_scale = pkg.cabi.conv2d_f16x3_split_weight(w, groups)
        # the one-pass split equals sdetr_split_f16_pair_dev of either layout, bit for bit
        for got, ref in (((f_hi, f_lo), w.permute(0, 2, 3, 1)), ((w_hi, w_lo), dgrad_weight(w, groups))):
            r_hi, r_lo, r_scale = pkg.cabi.split_f16_pair_dev(ref.contiguous(), w_scale)
            assert torch.equal(got[0], r_hi) and torch.equal(got[1], r_lo)
        dx = pkg.cabi.conv2d_f16x3_dgrad(gy, (ho, wo), pkg.cabi.pow2_scale(gbuf, 12), w_hi, w_lo, w_scale, groups, k, stride,
                                         (h, wd))
        dx = dx.double().transpose(1, 2).reshape(b, cin, h, wd)
        err = (dx - dx64).abs()
        assert bool((err <= 2.0 ** -17 * bdx + 1e-30).all()), (kind, b, h, wd, float(err.max()))


@pytest.mark.gpu
def test_upsample_backward_vs_fp64():
    gen = torch.Generator().manual_seed(5)
    for src, dst in [((13, 21), (25, 42)), ((7, 11), (20, 30)), ((1, 1), (3, 2)), ((50, 84), (100, 168))]:
        gbuf = torch.randn(2, dst[0] * dst[1] + 3, 2 * C, generator=gen).to(DEV)
        g = gbuf[:, 3:]
        got = pkg.cabi.upsample_nearest_concat_backward(g[:, :, :C], dst, src)
        x = torch.zeros(2, C, *src, dtype=torch.float64, requires_grad=True)
        (want,) = torch.autograd.grad(F.interpolate(x, size=dst, mode="nearest"), x,
                                      g[:, :, :C].double().cpu().transpose(1, 2).reshape(2, C, *dst))
        err = (got.double().cpu() - want.flatten(2).transpose(1, 2)).abs().max()
        assert err < 1e-5 * float(g.abs().max()) * (-(-dst[0] // src[0])) * (-(-dst[1] // src[1])), (src, dst, float(err))
        assert torch.equal(got, pkg.cabi.upsample_nearest_concat_backward(g[:, :, :C], dst, src))


# ---- GPU: module ------------------------------------------------------------------------------------------------------------
def _golden(name):
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return {k: (str(z[k]) if z[k].dtype.kind in "US" else torch.from_numpy(z[k])) for k in z.files}


def _net(dtype=torch.float32):
    g = _golden("neck_repnet.npz")
    net = pkg.RepVGGPluXNetwork([C] * 4, [C] * 4, groups=G, norm_layer=torch.nn.BatchNorm2d, activation=torch.nn.SiLU)
    net.load_state_dict(mng.neck_state_dict(json.loads(g["shapes_json"]), mng.NECK_SEED), strict=True)
    return net.to(DEV, dtype), g


def _maps(tok, shapes):
    b, _, c = tok.shape
    out, s = OrderedDict(), 0
    for i, (h, w) in enumerate(shapes):
        out[i] = tok[:, s:s + h * w].transpose(1, 2).reshape(b, c, h, w)
        s += h * w
    return out


def _torch_tokens(net, mem, shapes):
    return torch.cat([f.flatten(2).transpose(1, 2) for f in net(_maps(mem, shapes)).values()], 1)


class _NoTF32:
    def __enter__(self):
        self.prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.prev


def _step(net, mem, shapes, R, tokens):
    """one forward + backward of sum(out * R) -> (out, [grad(memory)] + parameter gradients)"""
    mem = mem.detach().clone().requires_grad_(True)
    out = net.forward_tokens(mem, shapes) if tokens else _torch_tokens(net, mem, shapes)
    params = [p for p in net.parameters()]
    grads = torch.autograd.grad((out * R).sum(), [mem] + params)
    return out.detach(), list(grads)


def _rel(a, ref):
    return float((a.detach().double() - ref.detach()).abs().max()) / max(float(ref.detach().abs().max()), 1e-30)


def _compare_vs_fp64(shapes, b, mode):
    """token path and fp32 forward() against a float64 forward() twin: outputs, gradients, updated running statistics"""
    net, g = _net()
    if shapes == mng.HALF_SHAPES and b == 2:
        mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous()
    else:
        gen = torch.Generator().manual_seed(7)
        mem = torch.randn(b, sum(h * w for h, w in shapes), C, generator=gen).to(DEV)
    R = torch.randn(mem.shape, generator=torch.Generator().manual_seed(8)).to(DEV)
    nets = {k: copy.deepcopy(net) for k in ("tok", "f32")}
    n64 = copy.deepcopy(net).double()
    for n in list(nets.values()) + [n64]:
        n.train(mode == "train")
    with _NoTF32():
        out, gr = _step(nets["tok"], mem, shapes, R, True)
        o32, g32 = _step(nets["f32"], mem, shapes, R, False)
        o64, g64 = _step(n64, mem.double(), shapes, R.double(), False)
    names = ["memory"] + [n for n, _ in net.named_parameters()]
    worst = 0.0
    for name, a, a32, a64 in zip(["out"] + names, [out] + gr, [o32] + g32, [o64] + g64):
        if name.endswith("conv_mask.bias"):
            continue  # the softmax is shift-invariant: the exact gradient is zero, both sides are round-off
        e, e32 = _rel(a, a64), _rel(a32, a64)
        worst = max(worst, e / (e32 + 1e-7))
        assert e <= FP32_MULTIPLE * e32 + 1e-7, (name, e, e32)
    sd, sd64 = nets["tok"].state_dict(), n64.state_dict()
    for k, v in nets["f32"].state_dict().items():
        if k.endswith(("running_mean", "running_var")):
            e, e32 = _rel(sd[k], sd64[k]), _rel(v, sd64[k])
            assert e <= FP32_MULTIPLE * e32 + 1e-7, (k, e, e32)
        elif k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v)
    print(f"{shapes[0]} b={b} {mode}: worst error / fp32 error = {worst:.2f}")
    return nets["tok"], out


@pytest.mark.gpu
def test_train_forward_tokens_matches_reference_fixture():
    """train-mode forward_tokens at HALF_SHAPES: the reference's train_rows and running statistics, within the tolerances of
    test_neck.py::test_torch_forward_matches_reference_eval_and_train"""
    net, g = _net()
    net.train()
    mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous()
    assert net.training_tokens_supported(mem, mng.HALF_SHAPES) and not net.tokens_supported(mem, mng.HALF_SHAPES)
    with torch.no_grad():
        out = net.forward_tokens(mem, mng.HALF_SHAPES)
    rows = torch.gather(out, 1, g["rows_index"].to(DEV)[..., None].expand(-1, -1, C)).cpu()
    assert (rows - g["train_rows"]).abs().max() < 1e-4 * max(1.0, float(g["train_rows"].abs().max()))
    sd = net.state_dict()
    for name in mng.TRAIN_STATS:
        for s in ("running_mean", "running_var"):
            assert (sd[f"{name}.{s}"].cpu() - g[f"train.{name}.{s}"]).abs().max() < 1e-5, (name, s)
        assert int(sd[f"{name}.num_batches_tracked"]) == int(g[f"train.{name}.num_batches_tracked"]) == 8


@pytest.mark.gpu
@pytest.mark.parametrize("shapes,b", [(mng.HALF_SHAPES, 2), (CONFIG2_SHAPES, 2), (mng.HALF_SHAPES, 1)])
def test_train_gradients_vs_fp64(shapes, b):
    _compare_vs_fp64(shapes, b, "train")


@pytest.mark.gpu
def test_eval_with_grad_matches_forward():
    net, _ = _compare_vs_fp64(mng.HALF_SHAPES, 2, "eval")
    mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous().requires_grad_(True)
    assert not net.tokens_supported(mem, mng.HALF_SHAPES) and net.training_tokens_supported(mem, mng.HALF_SHAPES)
    with torch.no_grad():
        assert net.tokens_supported(mem, mng.HALF_SHAPES) and not net.training_tokens_supported(mem, mng.HALF_SHAPES)


@pytest.mark.gpu
def test_sync_batchnorm_copy_matches():
    net, _ = _net()
    net.train()
    sync = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(net))
    mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous()
    assert sync.training_tokens_supported(mem, mng.HALF_SHAPES)
    R = torch.randn(mem.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    out, gr = _step(net, mem, mng.HALF_SHAPES, R, True)
    out_s, gr_s = _step(sync, mem, mng.HALF_SHAPES, R, True)
    assert torch.equal(out, out_s)
    for a, b in zip(gr, gr_s):
        assert torch.equal(a, b)
    for (k, v), (k2, v2) in zip(net.state_dict().items(), sync.state_dict().items()):
        assert k == k2 and torch.equal(v, v2), k


def _train_step_fn(net, mem, R):
    params = list(net.parameters())

    def step():
        out = net.forward_tokens(mem, mng.HALF_SHAPES)
        return [out] + list(torch.autograd.grad((out * R).sum(), [mem] + params))
    return step


@pytest.mark.gpu
def test_no_sync_constant_launches_and_graph_replay():
    net, _ = _net()
    net.train()
    mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous().requires_grad_(True)
    R = torch.randn(mem.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
    step = _train_step_fn(net, mem, R)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = step()
        counts = []
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in range(2):
                n0 = pkg.cabi.launch_count()
                again = step()
                counts.append(pkg.cabi.launch_count() - n0)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.current_stream().wait_stream(s)
    assert counts[0] == counts[1] > 0
    for a, b in zip(eager, again):
        assert torch.equal(a, b)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        static = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, static):
        assert torch.equal(a, b)
    print(f"library launches per forward + backward: {counts[0]}")


_DETERMINISM_SCRIPT = r"""
import sys, torch
sys.path[:0] = [ROOT, ROOT + "/tests"]
torch.use_deterministic_algorithms(True)
from test_neck_training import _net, _step, mng, DEV
import hashlib
net, _ = _net()
net.train()
mem = mng.tokens(mng.neck_inputs()).to(DEV).contiguous()
R = torch.randn(mem.shape, generator=torch.Generator().manual_seed(4)).to(DEV)
digests = []
for _ in range(2):
    n = __import__("copy").deepcopy(net)
    out, grads = _step(n, mem, mng.HALF_SHAPES, R, True)
    h = hashlib.sha256()
    for t in [out] + grads + list(n.buffers()):
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    digests.append(h.hexdigest())
print("DIGESTS", digests[0], digests[1])
"""


@pytest.mark.gpu
def test_deterministic_algorithms_bit_identical():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    code = "ROOT = %r\n" % ROOT + _DETERMINISM_SCRIPT
    res = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("DIGESTS")][0].split()
    assert line[1] == line[2]


# ---- GPU: transformer ------------------------------------------------------------------------------------------------------
def _transformer():
    torch.manual_seed(0)
    enc = pkg.SalienceTransformerEncoder(pkg.SalienceTransformerEncoderLayer(C, 64, 0.0, 8), 1, 40)
    neck, _ = _net()
    return pkg.SalienceTransformer(enc, neck, None).to(DEV)


def _transformer_inputs(shapes, b=2):
    gen = torch.Generator().manual_seed(1)
    feats = [torch.randn(b, C, h, w, generator=gen).to(DEV) for h, w in shapes]
    masks = [torch.zeros(b, h, w, dtype=torch.bool, device=DEV) for h, w in shapes]
    pos = [torch.randn(b, C, h, w, generator=gen).to(DEV) * 0.1 for h, w in shapes]
    return feats, masks, pos


@pytest.mark.gpu
def test_transformer_routes_training_neck_through_tokens(monkeypatch):
    """A training SalienceTransformer sends its RepVGG-PluX neck through forward_tokens (no NCHW route), and what the neck
    hands back -- its output, its parameter gradients, the gradient the encoder receives and the running statistics -- stays
    within FP32_MULTIPLE of a float64 twin of the neck run on the same encoder memory, as in the module tests.  The encoder
    itself has no float64 twin (its kernels are fp32-only); its backward is the same code on either route, fed by the
    gradient checked here."""
    shapes = [(16, 20), (8, 10), (4, 5), (2, 3)]
    tr = _transformer().train()
    feats, masks, pos = _transformer_inputs(shapes)
    # eager training keeps the NCHW route (the token step is host-bound there); while a CUDA graph is being captured the
    # transformer takes the token path -- the capture itself is checked at module level
    # (test_no_sync_constant_launches_and_graph_replay), here the capture state is stood in for
    ran = []
    monkeypatch.setattr(tr.neck, "forward_tokens", lambda *a: ran.append("tokens"))
    with torch.no_grad():
        tr.train()(feats, masks, pos)
    assert ran == []
    monkeypatch.undo()
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    tr.load_state_dict(_transformer().state_dict())  # the running statistics before any step
    calls, neck_in = [], []
    orig = tr.neck.forward_tokens
    monkeypatch.setattr(tr.neck, "forward_tokens", lambda m, s: calls.append(1) or neck_in.append(m) or orig(m, s))

    def no_nchw(*a, **k):
        raise AssertionError("the NCHW route ran")
    monkeypatch.setattr(tr.neck, "forward", no_nchw)
    monkeypatch.setattr(pkg.cabi, "tokens_to_maps", no_nchw)
    memory, _ = tr(feats, masks, pos)
    assert calls == [1] and neck_in[0].requires_grad
    R = torch.randn(memory.shape, generator=torch.Generator().manual_seed(2)).to(DEV)
    g_tok = torch.autograd.grad((memory * R).sum(), [neck_in[0]] + list(tr.neck.parameters()))
    monkeypatch.undo()
    assert not torch.cuda.is_current_stream_capturing()
    n32, _ = _net()  # the neck's state before the step
    n64 = copy.deepcopy(n32).double()
    with _NoTF32():
        o32, g32 = _step(n32.train(), neck_in[0], shapes, R, False)
        o64, g64 = _step(n64.train(), neck_in[0].double(), shapes, R.double(), False)
    names = ["out", "grad into the encoder"] + [n for n, _ in tr.neck.named_parameters()]
    for name, a, a32, a64 in zip(names, [memory] + list(g_tok), [o32] + g32, [o64] + g64):
        if name.endswith("conv_mask.bias"):
            continue  # the softmax is shift-invariant: the exact gradient is zero, both sides are round-off
        e, e32 = _rel(a, a64), _rel(a32, a64)
        assert e <= FP32_MULTIPLE * e32 + 1e-7, (name, e, e32)
    sd, sd32, sd64 = tr.neck.state_dict(), n32.state_dict(), n64.state_dict()
    for k in sd:
        if k.endswith(("running_mean", "running_var")):
            assert _rel(sd[k], sd64[k]) <= FP32_MULTIPLE * _rel(sd32[k], sd64[k]) + 1e-7, k
    # eval without autograd: the folded inference route, as before
    tr.eval()
    calls.clear()
    monkeypatch.setattr(tr.neck, "forward_tokens", lambda *a: calls.append(1) or orig(*a))
    with torch.no_grad():
        assert tr.neck.tokens_supported(memory.detach(), shapes)
        tr(feats, masks, pos)
    assert calls == [1]
