"""ResNetBackbone.forward_tokens under autograd (backbone.py, _TrainBlocks): the predicate, the torch mirror's gradients against
the UNMODIFIED reference (tests/golden/resnet50_backbone_grads.npz, made by tools/make_backbone_grad_golden.py) and the
backward chain's data flow with float64 stand-ins for the kernels, on the CPU; the input-gradient, weight-gradient and fold
kernels, the module's gradients, CUDA graphs and the backbone -> ChannelMapper chain on the GPU."""
import copy
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import salience_detr_b200 as pkg
from salience_detr_b200 import backbone as bbm
from salience_detr_b200 import cabi, synthetic
from conftest import GOLDEN
from tools import make_backbone_golden as mbg
from tools import make_backbone_grad_golden as mgg

DEV = "cuda:0"
FBN = pkg.FrozenBatchNorm2d


def _weights(arch="resnet50"):
    net = bbm.ResNet(**pkg.ResNetBackbone.model_arch[arch], norm_layer=FBN)
    return synthetic.resnet_weights({k: list(v.shape) for k, v in net.state_dict().items() if not k.startswith("fc.")},
                                    mbg.WEIGHT_SEED)


def _backbone(arch="resnet50", return_indices=(1, 2, 3), freeze_indices=(0,), **kw):
    return pkg.ResNetBackbone(arch, weights=_weights(arch), return_indices=return_indices, freeze_indices=freeze_indices,
                              norm_layer=kw.pop("norm_layer", FBN), **kw)


def _padded_images(b, H, W, gen):
    """b images in an (H, W) batch, image i of (H - 3 i, W - 5 i) pixels and zero padding"""
    x = torch.zeros(b, 3, H, W)
    for i in range(b):
        h, w = max(1, H - 3 * i), max(1, W - 5 * i)
        x[i, :, :h, :w] = torch.randn(3, h, w, generator=gen)
    return x


def _loss(outs, cot):
    return sum((v * cot[k]).sum() for k, v in outs.items())


def _cotangents(shapes, seed, device="cpu", dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(s, generator=g, dtype=torch.float64).to(device, dtype) for k, s in shapes.items()}


def _trainable(m):
    return [(n, p) for n, p in m.named_parameters() if p.requires_grad]


# ---- CPU: predicate -----------------------------------------------------------------------------------------------------
def test_training_tokens_supported_cases(monkeypatch):
    m = _backbone()
    x = torch.randn(1, 3, 32, 32)
    with torch.enable_grad():
        assert not m.training_tokens_supported(x)  # CPU
    # the rest on CPU parameters and a CPU image taken for a CUDA one
    monkeypatch.setattr(bbm, "_cuda_image", lambda t: True)
    assert m.layers_supported()
    with torch.enable_grad():
        assert m.training_tokens_supported(x)
        assert not m.tokens_supported(x)  # a parameter requires a gradient: inference does not hold
        assert not m.training_tokens_supported(x.clone().requires_grad_(True))  # an image gradient
        assert _backbone(freeze_indices=(2,)).training_tokens_supported(x)  # a frozen stage in the middle: trains through it
        assert _backbone(freeze_indices=(0, 1)).training_tokens_supported(x)
        assert not _backbone(freeze_indices=(0, 1, 2, 3)).training_tokens_supported(x)  # nothing trains
        stem = _backbone(freeze_indices=())  # a trainable stem
        assert stem.conv1.weight.requires_grad and not stem.training_tokens_supported(x)
        assert not pkg.ResNetBackbone("resnet18", norm_layer=FBN, freeze_indices=(0,)).training_tokens_supported(x)
        assert not pkg.ResNetBackbone("resnet50", freeze_indices=(0,)).training_tokens_supported(x)  # nn.BatchNorm2d
        assert not pkg.ResNetBackbone("resnext50_32x4d", norm_layer=FBN, freeze_indices=(0,)).training_tokens_supported(x)
    with torch.no_grad():
        assert not m.training_tokens_supported(x)  # no autograd
    with torch.enable_grad():
        assert not copy.deepcopy(m).half().training_tokens_supported(x)  # fp16 parameters


def test_forward_tokens_still_raises_when_neither_holds():
    m = _backbone()
    with torch.enable_grad(), pytest.raises(RuntimeError, match="needs forward"):
        m.forward_tokens(torch.randn(1, 3, 32, 32))


# ---- CPU: the torch mirror against the reference -------------------------------------------------------------------------
def test_mirror_gradients_match_reference_fixture():
    z = np.load(os.path.join(GOLDEN, "resnet50_backbone_grads.npz"), allow_pickle=False)
    names = json.loads(str(z["names_json"]))
    m = _backbone().double()
    assert [n for n, _ in _trainable(m)] == names and len(names) == 42
    stats = mgg.gradient_stats(m, mbg.image().double())
    for i, n in enumerate(names):
        sumsq, dot = stats[n]
        assert abs(sumsq - z["sumsq"][i]) <= 1e-9 * z["sumsq"][i], n
        numel = dict(m.named_parameters())[n].numel()
        assert abs(dot - z["dot"][i]) <= 1e-9 * (z["sumsq"][i] * numel) ** 0.5, n


# ---- CPU: the backward chain's data flow with float64 stand-ins ------------------------------------------------------------
def _tok(x):
    b, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(b, h * w, c)


def _nchw(t, hw):
    b, _, c = t.shape
    return t.reshape(b, hw[0], hw[1], c).permute(0, 3, 1, 2)


class _Float64Kernels:
    """the cabi calls of the training path restated in float64 torch, counting the library launches each one stands for"""

    def __init__(self):
        self.launches = 0
        self.calls = []

    def _n(self, k):
        self.launches += k

    def frozen_bn_fold(self, w, bn, scale=True, bias=True):
        self._n(1)
        s = bn.weight.double() * (bn.running_var.double() + bn.eps).rsqrt()
        return w.double() * s.view(-1, *[1] * (w.dim() - 1)), s, bn.bias.double() - bn.running_mean.double() * s

    def conv2d_f16x3_split_weight(self, w, groups, dgrad=True):
        self._n(2)  # the weight's scale and the split
        return w, w, w if dgrad else None, w if dgrad else None, torch.ones(1, dtype=torch.float64)

    def resnet_stem(self, x, w, b):
        self._n(1)
        return _tok(F.relu(F.conv2d(x.double(), w.t().reshape(64, 3, 7, 7), b, 2, 3)))

    def maxpool3x3s2_tokens(self, t, hw):
        self._n(1)
        return _tok(F.max_pool2d(_nchw(t, hw), 3, 2, 1))

    def pow2_scale(self, x, target=12):
        self._n(1)
        return torch.ones(1, dtype=torch.float64)

    def conv2d_f16x3(self, x, hw, a_scale, w_hi, w_lo, w_scale, bias, groups, ksize, stride, act=0, out=None, z=None):
        self._n(1)
        y = _tok(F.conv2d(_nchw(x, hw), w_hi, bias, stride, ksize // 2))
        y = y + z if z is not None else y
        y = F.relu(y) if act == cabi.ACT_RELU else y
        return out.copy_(y) if out is not None else y.contiguous()

    def conv2d_f16x3_dgrad(self, dy, dy_hw, a_scale, w_hi, w_lo, w_scale, groups, ksize, stride, hw, z=None, m=None, out=None):
        self._n(1)
        self.calls.append(("dgrad", tuple(w_hi.shape), stride, z is not None, m is not None, out is not None and out is z))
        b = dy.shape[0]
        dx = _tok(torch.nn.grad.conv2d_input((b, w_hi.shape[1], hw[0], hw[1]), w_hi, _nchw(dy, dy_hw), stride, ksize // 2))
        dx = dx + z if z is not None else dx
        dx = torch.ops.aten.threshold_backward(dx, m, 0) if m is not None else dx
        return out.copy_(dx) if out is not None else dx.contiguous()

    def conv2d_f16x3_wgrad(self, dy, dy_scale, x, x_scale, hw, weight_shape, stride, cout_scale=None):
        self._n(2)
        self.calls.append(("wgrad", tuple(weight_shape), stride))
        k = weight_shape[-1]
        ho, wo = ((v + 2 * (k // 2) - k) // stride + 1 for v in hw)
        dw = torch.nn.grad.conv2d_weight(_nchw(x, hw), weight_shape, _nchw(dy, (ho, wo)), stride, k // 2)
        return dw * cout_scale.view(-1, 1, 1, 1) if cout_scale is not None else dw


FLOW_CASES = {
    "r50_f0_r123": ("resnet50", (0,), (1, 2, 3)),
    "r50_f0_r0123": ("resnet50", (0,), (0, 1, 2, 3)),
    "r50_f01": ("resnet50", (0, 1), (1, 2, 3)),
    "r50_f2_middle": ("resnet50", (2,), (1, 2, 3)),
    "r50_f0_r02": ("resnet50", (0,), (0, 2)),
}


@pytest.mark.parametrize("case", sorted(FLOW_CASES))
def test_backward_chain_data_flow_float64(case, monkeypatch):
    """_train_tokens with every kernel replaced by its float64 torch statement gives forward()'s outputs and gradients in
    float64 (masks, residual sums, FrozenBatchNorm scales, returned maps' gradients), and the stand-ins count
    launches_per_training_step() launches"""
    arch, freeze, ret = FLOW_CASES[case]
    m = _backbone(arch, return_indices=ret, freeze_indices=freeze).double()
    # non-trivial FrozenBatchNorm statistics, so a missing or doubled scale shows
    gen = torch.Generator().manual_seed(7)
    for mod in m.modules():
        if isinstance(mod, FBN):
            c = mod.weight.numel()
            mod.weight.copy_(torch.rand(c, generator=gen, dtype=torch.float64) + 0.5)
            mod.running_var.copy_(torch.rand(c, generator=gen, dtype=torch.float64) + 0.5)
    x = _padded_images(2, 61, 83, torch.Generator().manual_seed(8)).double()
    fake = _Float64Kernels()
    for name in ("frozen_bn_fold", "conv2d_f16x3_split_weight", "resnet_stem", "maxpool3x3s2_tokens", "pow2_scale",
                 "conv2d_f16x3", "conv2d_f16x3_dgrad", "conv2d_f16x3_wgrad"):
        monkeypatch.setattr(cabi, name, getattr(fake, name))
    ref_m = copy.deepcopy(m)
    ref = ref_m(x)
    cot = _cotangents({k: v.shape for k, v in ref.items()}, 9, dtype=torch.float64)
    ref_g = torch.autograd.grad(_loss(ref, cot), [p for _, p in _trainable(ref_m)])
    outs = m._train_tokens(x)
    assert list(outs) == list(ref)
    for k in ref:
        assert float((outs[k] - ref[k]).detach().abs().max()) <= 1e-12 * float(ref[k].abs().max()), k
    _loss(outs, cot).backward()
    assert fake.launches == m.launches_per_training_step()
    for (n, p), g in zip(_trainable(m), ref_g):
        assert p.grad is not None, n
        assert float((p.grad - g).abs().max()) <= 1e-10 * float(g.abs().max()), n
    assert all(p.grad is None for p in m.parameters() if not p.requires_grad)
    # below the first trainable block, each block input's gradient is one masked input gradient written over its residual
    # operand; the first trainable block computes none
    blocks, first, _ = m._train_plan()
    assert sum(1 for c in fake.calls if c[0] == "dgrad" and c[3] and c[4] and c[5]) == len(blocks) - first - 1
    assert sum(1 for c in fake.calls if c[0] == "wgrad") == len(_trainable(m))


def test_launches_per_training_step_resnet50():
    m = _backbone()
    # forward: stem fold, stem, max-pool, 3 per convolution (52), 6 per block (16) + 4 downsamples
    fwd = 3 + 3 * 52 + 6 * 16 + 4
    # backward over layers 2-4 (13 blocks, 3 downsamples): G's scale, 2 input gradients + 2 scales, 3 weight gradients of 2
    # launches, the downsample's weight gradient, and below the first block the block input's gradient (+ the downsample's)
    bwd = 13 * (1 + 4 + 6) + 3 * 2 + 12 * 1 + 2
    assert m.launches_per_training_step() == fwd + bwd == 422


# ---- GPU: kernels ---------------------------------------------------------------------------------------------------------
def _dgrad_ref(dy, w, hw, stride):
    """float64 input gradient (NCHW) of conv(x, w) at stride, padding k // 2, dy NCHW"""
    b = dy.shape[0]
    return torch.nn.grad.conv2d_input((b, w.shape[1], hw[0], hw[1]), w.double(), dy.double(), stride, w.shape[-1] // 2)


@pytest.mark.gpu
@pytest.mark.parametrize("k,stride,cin,cout", [(1, 1, 256, 64), (3, 1, 64, 64), (3, 2, 128, 128), (1, 2, 256, 512),
                                               (1, 1, 64, 256)])
@pytest.mark.parametrize("hw", [(13, 21), (1, 1), (7, 3)])
@pytest.mark.parametrize("mode", ["plain", "z", "z_alias", "mask", "z_mask_alias"])
def test_dgrad_vs_fp64(k, stride, cin, cout, hw, mode):
    """dx = conv^T(dy, W) (+ z), 0 where m <= 0: within the forward convolution's bound 2^-17 * (|dy| conv^T |W|) + |z|
    rounding; where m <= 0 exactly 0, where m is NaN or > 0 the value passes, a NaN value stays NaN"""
    gen = torch.Generator().manual_seed(k * 1000 + stride * 100 + cin + cout + hw[0] * 7 + hw[1] + len(mode))
    b, (h, w) = 2, hw
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    wt = torch.randn(cout, cin, k, k, generator=gen) / (cin * k * k) ** 0.5
    dy = torch.randn(b, cout, ho, wo, generator=gen)
    z = torch.randn(b, cin, h, w, generator=gen)
    msrc = torch.randn(b, cin, h, w, generator=gen)
    msrc[msrc.abs() < 0.3] = 0.0
    msrc.view(-1)[::97] = float("nan")
    f_hi, f_lo, d_hi, d_lo, ws = cabi.conv2d_f16x3_split_weight(wt.to(DEV), 1, True)
    dyr = _tok(dy).contiguous().to(DEV)
    s = cabi.pow2_scale(dyr, 12)
    ref = _dgrad_ref(dy, wt, (h, w), stride)
    bnd = _dgrad_ref(dy.abs(), wt.abs(), (h, w), stride)
    zr, mr = _tok(z).contiguous().to(DEV), _tok(msrc).contiguous().to(DEV)
    kw = {}
    if mode in ("z", "z_alias", "z_mask_alias"):
        ref, bnd = ref + z.double(), bnd + z.double().abs()
        kw["z"] = zr
    if mode in ("z_alias", "z_mask_alias"):
        kw["out"] = zr
    if mode in ("mask", "z_mask_alias"):
        kw["m"] = mr
        ref = torch.ops.aten.threshold_backward(ref, msrc.double(), 0)
    zc = zr.clone()
    got = cabi.conv2d_f16x3_dgrad(dyr, (ho, wo), s, d_hi, d_lo, ws, 1, k, stride, (h, w), **kw)
    if mode == "z":
        assert torch.equal(zr, zc)
    if "out" in kw:
        assert got is zr
    got = _nchw(got.cpu().double(), (h, w))
    if "m" in kw:
        dead = msrc <= 0
        assert bool((got[dead] == 0).all()) and bool(dead.any()) and bool(msrc.isnan().any())
    assert bool(((got - ref).abs() <= 2.0 ** -17 * bnd + 1e-30).all()), float((got - ref).abs().max())


@pytest.mark.gpu
def test_dgrad_mask_nan_rules():
    """torch's threshold_backward: a NaN mask source lets the value through, a NaN value stays NaN (unless masked)"""
    cin = cout = 64
    wt = torch.zeros(cout, cin, 1, 1)
    wt[:, :, 0, 0] = torch.eye(64)
    f_hi, f_lo, d_hi, d_lo, ws = cabi.conv2d_f16x3_split_weight(wt.to(DEV), 1, True)
    dy = torch.ones(1, 4, 64)
    dy[0, 1, :] = float("nan")
    dy = dy.to(DEV)
    msrc = torch.tensor([1.0, 1.0, -1.0, float("nan")]).view(1, 4, 1).expand(1, 4, 64).contiguous().to(DEV)
    s = torch.ones(1, device=DEV)
    got = cabi.conv2d_f16x3_dgrad(dy, (2, 2), s, d_hi, d_lo, ws, 1, 1, 1, (2, 2), m=msrc).cpu()
    assert bool((got[0, 0] == 1).all()) and bool(got[0, 1].isnan().all()) and bool((got[0, 2] == 0).all())
    assert bool((got[0, 3] == 1).all())


@pytest.mark.gpu
@pytest.mark.parametrize("k,c", [(3, 64), (1, 256), (3, 256), (1, 64), (3, 128)])
def test_stride1_dgrad_is_the_forward_on_flipped_weights(k, c):
    """z = m = NULL, stride 1: the bits of sdetr_conv2d_f16x3 on dY with the flipped weights"""
    gen = torch.Generator().manual_seed(k + 10 + c)
    b, h, w = 2, 50, 84
    wt = (torch.randn(c, c, k, k, generator=gen) / (c * k * k) ** 0.5).to(DEV)
    dy = torch.randn(b, h * w, c, generator=gen).to(DEV)
    _, _, d_hi, d_lo, ws = cabi.conv2d_f16x3_split_weight(wt, 1, True)
    s = cabi.pow2_scale(dy, 12)
    dgrad = cabi.conv2d_f16x3_dgrad(dy, (h, w), s, d_hi, d_lo, ws, 1, k, 1, (h, w))
    forward = cabi.conv2d_f16x3(dy, (h, w), s, d_hi, d_lo, ws, None, 1, k, 1, 0)
    assert torch.equal(forward, dgrad)


@pytest.mark.gpu
@pytest.mark.parametrize("k,stride,cin,cout", [(1, 1, 64, 256), (3, 2, 128, 128), (1, 2, 256, 512)])
def test_wgrad_scale_is_the_scaled_unscaled_result(k, stride, cin, cout):
    gen = torch.Generator().manual_seed(k + stride + cin + cout)
    b, h, w = 2, 29, 37
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    x = torch.randn(b, h * w, cin, generator=gen).to(DEV)
    dy = torch.randn(b, ho * wo, cout, generator=gen).to(DEV)
    sc = (torch.rand(cout, generator=gen) * 3 + 0.01).to(DEV)
    xs, ds = cabi.pow2_scale(x, 12), cabi.pow2_scale(dy, 12)
    plain = cabi.conv2d_f16x3_wgrad(dy, ds, x, xs, (h, w), (cout, cin, k, k), stride)
    scaled = cabi.conv2d_f16x3_wgrad(dy, ds, x, xs, (h, w), (cout, cin, k, k), stride, cout_scale=sc)
    again = cabi.conv2d_f16x3_wgrad(dy, ds, x, xs, (h, w), (cout, cin, k, k), stride, cout_scale=sc)
    assert torch.equal(scaled, plain * sc.view(-1, 1, 1, 1)) and torch.equal(scaled, again)
    ref = torch.nn.grad.conv2d_weight(_nchw(x.cpu().double(), (h, w)), (cout, cin, k, k), _nchw(dy.cpu().double(), (ho, wo)),
                                      stride, k // 2) * sc.cpu().double().view(-1, 1, 1, 1)
    assert float((scaled.cpu().double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


def _fold(conv, bn):
    """(W * scale, bias - running_mean * scale) in float64 torch, scale = weight * rsqrt(running_var + eps)"""
    scale = bn.weight.double() * (bn.running_var.double() + bn.eps).rsqrt()
    return conv.weight.double() * scale.view(-1, 1, 1, 1), bn.bias.double() - bn.running_mean.double() * scale


@pytest.mark.gpu
def test_device_fold_is_the_float64_fold():
    m = _backbone().to(DEV)
    for conv, bn in ((m.conv1, m.bn1), (m.layer3[1].conv2, m.layer3[1].bn2), (m.layer4[0].downsample[0], m.layer4[0].downsample[1])):
        bn.running_var.mul_(torch.rand_like(bn.running_var) + 0.5)
        w, b = _fold(conv, bn)
        wf, s, bf = cabi.frozen_bn_fold(conv.weight.detach(), bn)
        s64 = bn.weight.double() * (bn.running_var.double() + bn.eps).rsqrt()
        assert torch.equal(wf, w.float()) and torch.equal(bf, b.float()) and torch.equal(s, s64.float())


# ---- GPU: the module ------------------------------------------------------------------------------------------------------
def _torch_grads(m, x, cot, dtype=None, tf32=False):
    """forward()'s outputs and trainable gradients: float64 when dtype is float64, else cuDNN fp32 with TF32 on or off"""
    mm = copy.deepcopy(m)
    xx = x
    if dtype is not None:
        mm, xx = mm.to(dtype), x.to(dtype)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        outs = mm(xx)  # a parameter requires a gradient: forward() is the torch chain
        grads = torch.autograd.grad(_loss(outs, {k: v.to(xx.dtype) for k, v in cot.items()}), [p for _, p in _trainable(mm)])
    finally:
        torch.backends.cudnn.allow_tf32 = old
    return outs, grads


def _rel(got, ref):
    return float((got.double() - ref.double()).abs().max()) / float(ref.double().abs().max())


class _ExactBackward:
    """the backward's kernels (input and weight gradients) replaced by float64 torch on the same operands: the exact backward
    through the token forward's own activations and ReLU masks"""
    NAMES = ("conv2d_f16x3_dgrad", "conv2d_f16x3_wgrad")

    def __enter__(self):
        f64 = _Float64Kernels()
        self.saved = {n: getattr(cabi, n) for n in self.NAMES}

        def dgrad(dy, dy_hw, a_scale, d_hi, d_lo, ws, groups, ks, stride, hw, z=None, m=None, out=None):
            w = ((d_hi.double() + d_lo.double()) / ws.double()).permute(3, 0, 1, 2).flip(2, 3)  # W' -> W, exactly
            r = f64.conv2d_f16x3_dgrad(dy.double(), dy_hw, None, w, None, None, groups, ks, stride, hw,
                                       z=z.double() if z is not None else None, m=m.double() if m is not None else None).float()
            return out.copy_(r) if out is not None else r

        def wgrad(dy, dy_scale, x, x_scale, hw, shape, stride, cout_scale=None):
            return f64.conv2d_f16x3_wgrad(dy.double(), None, x.double(), None, hw, shape, stride,
                                          cout_scale=cout_scale.double() if cout_scale is not None else None).float()

        cabi.conv2d_f16x3_dgrad, cabi.conv2d_f16x3_wgrad = dgrad, wgrad
        return self

    def __exit__(self, *exc):
        for n, f in self.saved.items():
            setattr(cabi, n, f)


MODULE_CASES = {
    "r50_small": ("resnet50", (0,), (1, 2, 3), 1, 64, 96),
    "r50_ragged": ("resnet50", (0,), (1, 2, 3), 3, 120, 168),
    "r50_config2": ("resnet50", (0,), (1, 2, 3), 2, 800, 1344),
    "r50_r0123": ("resnet50", (0,), (0, 1, 2, 3), 2, 97, 131),
    "r50_f01": ("resnet50", (0, 1), (1, 2, 3), 2, 97, 131),
    "r50_f2": ("resnet50", (2,), (1, 2, 3), 2, 97, 131),
    "wide50": ("wide_resnet50_2", (0,), (1, 2, 3), 1, 97, 131),
    "r101": ("resnet101", (0,), (1, 2, 3), 2, 64, 96),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(MODULE_CASES))
def test_training_tokens_vs_fp64(case):
    """outputs bit-identical to no_grad forward_tokens; every trainable weight's gradient within 16x the error of forward()
    on cuDNN fp32 (TF32 off) against float64, and below TF32's, measured against the float64 backward through the token
    forward's own ReLU masks; frozen parameters get none.

    Against forward() in float64 directly, a gradient also carries the forward's ReLU decisions: a pre-activation within the
    forward's rounding of zero takes the other branch, and a whole pixel's gradient changes with it.  At these map sizes
    (layer 3 is 4 x 6 at 64 x 96) one such pixel moves a weight gradient by 1e-3 to 1e-2 relative; cuDNN fp32 flips other
    pixels, or none.  That error is the inference forward's and is printed, not bounded here."""
    arch, freeze, ret, b, H, W = MODULE_CASES[case]
    m = _backbone(arch, return_indices=ret, freeze_indices=freeze).to(DEV)
    x = _padded_images(b, H, W, torch.Generator().manual_seed(H + W)).to(DEV)
    with torch.no_grad():
        inf = m.forward_tokens(x)
    assert m.training_tokens_supported(x)
    cot = _cotangents({k: v.shape for k, v in inf.items()}, 5, DEV)
    outs = m.forward_tokens(x)
    for k in inf:
        assert torch.equal(outs[k], inf[k]) and outs[k].stride() == inf[k].stride(), k
    grads = torch.autograd.grad(_loss(outs, cot), [p for _, p in _trainable(m)])
    with _ExactBackward():
        exact = torch.autograd.grad(_loss(m.forward_tokens(x), cot), [p for _, p in _trainable(m)])
    _, g64 = _torch_grads(m, x, cot, torch.float64)
    _, g32 = _torch_grads(m, x, cot)
    _, gtf = _torch_grads(m, x, cot, tf32=True)
    worst, direct = 0.0, 0.0
    for (n, _), g, ex, r, a, t in zip(_trainable(m), grads, exact, g64, g32, gtf):
        e, e32, etf = _rel(g, ex), _rel(a, r), _rel(t, r)
        worst, direct = max(worst, e / e32), max(direct, _rel(g, r))
        assert e <= 16 * e32 and e < etf, (n, e, e32, etf)
    print(f"{case}: worst backward error / cuDNN fp32's = {worst:.2f}; worst error against forward() in float64 {direct:.2e}, "
          f"cuDNN fp32 {max(_rel(a, r) for a, r in zip(g32, g64)):.2e}, TF32 {max(_rel(t, r) for t, r in zip(gtf, g64)):.2e}")
    m.zero_grad(set_to_none=True)
    _loss(m.forward_tokens(x), cot).backward()
    assert all((p.grad is not None) == p.requires_grad for p in m.parameters())


@pytest.mark.gpu
def test_train_and_eval_mode_agree_and_two_backwards_same_bits():
    m = _backbone().to(DEV)
    x = _padded_images(2, 97, 131, torch.Generator().manual_seed(1)).to(DEV)
    res = []
    for mode in (True, False, True):
        m.train(mode)
        outs = m.forward_tokens(x)
        cot = _cotangents({k: v.shape for k, v in outs.items()}, 2, DEV)
        res.append((outs, torch.autograd.grad(_loss(outs, cot), [p for _, p in _trainable(m)])))
    for outs, grads in res[1:]:
        assert all(torch.equal(outs[k], res[0][0][k]) for k in outs)
        assert all(torch.equal(a, b) for a, b in zip(grads, res[0][1]))


@pytest.mark.gpu
def test_no_sync_launch_count_and_channels_last_or_strided_gradients():
    m = _backbone(return_indices=(0, 1, 2, 3)).to(DEV)
    x = _padded_images(2, 97, 131, torch.Generator().manual_seed(3)).to(DEV)
    outs = m.forward_tokens(x)
    cot = _cotangents({k: v.shape for k, v in outs.items()}, 4, DEV)
    want = torch.autograd.grad(_loss(outs, cot), [p for _, p in _trainable(m)])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = cabi.launch_count()
        outs = m.forward_tokens(x)
        # cotangents as channels-last tensors (read in place) and as NCHW ones (one copy each)
        cl = {k: v.contiguous(memory_format=torch.channels_last) for k, v in cot.items()}
        got = torch.autograd.grad(_loss(outs, cl), [p for _, p in _trainable(m)])
        assert cabi.launch_count() - n0 == m.launches_per_training_step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all(torch.equal(a, b) for a, b in zip(got, want))


@pytest.mark.gpu
def test_cuda_graph_step_with_sgd_equals_eager():
    """forward + backward + an SGD step captured in one CUDA graph and replayed: each replay equals the same eager step bit for
    bit, the weights moving in place between replays (no per-version cache on this path)"""
    m_graph = _backbone().to(DEV)
    m_eager = copy.deepcopy(m_graph)
    x = _padded_images(2, 97, 131, torch.Generator().manual_seed(6)).to(DEV)
    with torch.no_grad():
        shapes = {k: v.shape for k, v in m_eager.forward_tokens(x).items()}
    cot = _cotangents(shapes, 7, DEV)
    # a learning rate that moves the weights by about 1e-3 of their size per step
    g0 = torch.autograd.grad(_loss(m_eager.forward_tokens(x), cot), [p for _, p in _trainable(m_eager)])
    lr = 1e-3 * max(float(p.abs().max()) for _, p in _trainable(m_eager)) / max(float(g.abs().max()) for g in g0)
    opt_g = torch.optim.SGD([p for _, p in _trainable(m_graph)], lr=lr)
    opt_e = torch.optim.SGD([p for _, p in _trainable(m_eager)], lr=lr)

    def step(m, opt):
        opt.zero_grad(set_to_none=False)
        loss = _loss(m.forward_tokens(x), cot)
        loss.backward()
        opt.step()
        return loss.detach()

    for _, p in _trainable(m_graph):
        p.grad = torch.zeros_like(p)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        probe = copy.deepcopy(m_graph)
        po = torch.optim.SGD([p for _, p in _trainable(probe)], lr=lr)
        for _, p in _trainable(probe):
            p.grad = torch.zeros_like(p)
        step(probe, po)  # warms up the library outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_loss = step(m_graph, opt_g)
    for _, p in _trainable(m_eager):
        p.grad = torch.zeros_like(p)
    for it in range(3):
        graph.replay()
        e_loss = step(m_eager, opt_e)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(e_loss)) and torch.equal(g_loss, e_loss), it
        for (n, a), (_, b) in zip(_trainable(m_graph), _trainable(m_eager)):
            assert torch.equal(a, b), (it, n)
        with torch.no_grad():  # an in-place update between replays that no optimizer state knows about
            m_graph.layer3[0].conv2.weight.mul_(0.99)
            m_eager.layer3[0].conv2.weight.mul_(0.99)


@pytest.mark.gpu
def test_backbone_channel_mapper_loss_chain():
    """backbone (token training) -> ChannelMapper (torch, training) -> loss: the backbone's weight gradients within the bound
    of test_training_tokens_vs_fp64 (against the float64 backward through the token forward), the all-torch chain giving the
    fp32 and float64 references"""
    bb = _backbone().to(DEV)
    torch.manual_seed(11)
    mapper = pkg.ChannelMapper([512, 1024, 2048], 256, 4).to(DEV).train()
    x = _padded_images(2, 97, 131, torch.Generator().manual_seed(12)).to(DEV)

    def run(b, mp, xx, tokens):
        feats = b.forward_tokens(xx) if tokens else b(xx)
        assert tokens or not b.tokens_supported(xx)
        outs = mp(feats)
        g = torch.Generator().manual_seed(13)
        loss = sum((o * torch.randn(o.shape, generator=g, dtype=torch.float64).to(o.device, o.dtype)).sum() for o in outs)
        return torch.autograd.grad(loss, [p for _, p in _trainable(b)])

    got = run(bb, mapper, x, True)
    with _ExactBackward():
        exact = run(bb, mapper, x, True)
    ref = run(copy.deepcopy(bb).double(), copy.deepcopy(mapper).double(), x.double(), False)
    old = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = False
        fp32 = run(copy.deepcopy(bb), copy.deepcopy(mapper), x, False)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    for (n, _), g, ex, r, a in zip(_trainable(bb), got, exact, ref, fp32):
        assert _rel(g, ex) <= 16 * _rel(a, r), (n, _rel(g, ex), _rel(a, r))
