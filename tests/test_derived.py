"""Derived-weight caches (derived.py): ``derived.cached`` and every method built on it return the same object while the source
tensors are unchanged, and a new value, equal to one built from scratch, after a source is modified in place, replaced by a
tensor whose version counter is equal, or has its ``.data`` swapped for another view of the same storage."""
import copy
import gc
from functools import reduce

import numpy as np
import pytest
import torch
from torch import nn

import salience_detr_b200 as pkg
from salience_detr_b200 import derived

DEV = "cuda:0"
CHANGES = ["in_place", "replaced", "data_view"]


def _equal(a, b) -> bool:
    if isinstance(a, (tuple, list)):
        return type(a) is type(b) and len(a) == len(b) and all(map(_equal, a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal(a[k], b[k]) for k in a)
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    if hasattr(a, "__dict__"):  # neck.py's TokenConv / _KGate
        return type(a) is type(b) and _equal(vars(a), vars(b))
    return a == b


def _swap_to_view(t):
    """t.data <- another view of t's storage with t's shape: the transpose of dims 0 and 1 (square in them), or for a vector a
    broadcast of its first element"""
    assert t.dim() == 1 or t.shape[0] == t.shape[1]
    t.data = t.data.transpose(0, 1) if t.dim() > 1 else t.data.as_strided(t.shape, (0,))


def _check_site(owner, read, replaced: str, viewed: str, change: str):
    """``read(owner)`` is cached, then rebuilt after ``change`` to the source at the dotted path ``replaced`` (for "replaced")
    or ``viewed`` (for "in_place" and "data_view"); the new value equals ``read`` of a fresh copy of the owner"""
    with torch.no_grad():
        for p in owner.parameters():
            p.uniform_(-1.0, 1.0)  # no zero-initialised weight: a stale value must differ from a fresh one
    *path, attr = (replaced if change == "replaced" else viewed).split(".")
    parent = reduce(getattr, path, owner)
    src = getattr(parent, attr)
    if change == "replaced":
        new = torch.empty_like(src).uniform_(0.5, 1.5)
        new = nn.Parameter(new, src.requires_grad) if isinstance(src, nn.Parameter) else new
        with torch.no_grad():
            for a, b in ((new, src), (src, new)):  # level the version counters before the first read
                while a._version < b._version:
                    a.mul_(1.0)
        assert new._version == src._version
    v0 = read(owner)
    assert read(owner) is v0
    with torch.no_grad():
        if change == "in_place":
            src.add_(1.0)
        elif change == "replaced":
            setattr(parent, attr, new)
        else:
            ptr, version, shape = src.data_ptr(), src._version, src.shape
            _swap_to_view(src)
            assert (src.data_ptr(), src._version, src.shape) == (ptr, version, shape)
    v1 = read(owner)
    assert v1 is not v0 and _equal(v1, read(copy.deepcopy(owner)))
    assert read(owner) is v1


# ---- the helper --------------------------------------------------------------------------------------------------------
def test_hit_returns_the_same_object_and_builds_once():
    w = torch.randn(6, 6, requires_grad=True)
    calls = []

    def build():
        calls.append(1)
        return w * 2

    a = derived.cached(w, "double", (w,), build)
    assert derived.cached(w, "double", (w,), build) is a and len(calls) == 1
    assert not a.requires_grad  # build() runs without autograd
    assert derived.cached(w, "other", (w,), lambda: w * 3) is not a  # one entry per name


@pytest.mark.parametrize("change", CHANGES)
def test_helper_rebuilds_after_a_source_changes(change):
    lin = nn.Linear(8, 8)
    _check_site(lin, lambda m: derived.cached(m, "t", (m.weight, m.bias), lambda: (m.weight.t().contiguous(), m.bias * 1)),
                "weight", "weight", change)


def test_freed_owners_leave_no_entries():
    gc.collect()
    n = len(derived._entries)
    for _ in range(200):
        w = torch.randn(4, 4)
        derived.cached(w, "t", (w,), lambda: w.t().contiguous())
    for make, read, _, _ in CPU_SITES.values():  # no cached value may hold its owner alive
        read(make())
    del w
    gc.collect()
    assert len(derived._entries) == n


# ---- the sites reachable on the CPU ------------------------------------------------------------------------------------
def _encoder_layer():
    return pkg.SalienceTransformerEncoderLayer(64, 128, 0.0, 2, topk_sa=20)


def _encoder():
    return pkg.SalienceTransformerEncoder(_encoder_layer(), 2, 40)


# site: (make the owner, read the derived value, source replaced by one of equal version, source given a new view)
CPU_SITES = {
    "MaskPredictor.transposed_weights": (lambda: pkg.MaskPredictor(256, 256), lambda m: m.transposed_weights(),
                                         "layer2.4.bias", "layer1.1.weight"),
    "SalienceTransformerEncoderLayer._mha_views": (_encoder_layer, lambda m: m._mha_views(), "pre_attention.in_proj_bias",
                                                   "pre_attention.in_proj_bias"),
    "SalienceTransformerEncoderLayer._mha_transposed": (_encoder_layer, lambda m: m._mha_transposed(),
                                                        "pre_attention.in_proj_weight", "pre_attention.out_proj.weight"),
    "SalienceTransformerEncoder._value_projection": (_encoder, lambda m: m._value_projection(),
                                                     "layers.1.self_attn.value_proj.bias", "layers.0.self_attn.value_proj.weight"),
    "SalienceTransformerDecoder._value_projection": (
        lambda: pkg.SalienceTransformerDecoder(pkg.SalienceTransformerDecoderLayer(64, 128, 2, 0.0), 2, 11),
        lambda m: m._value_projection(), "layers.1.cross_attn.value_proj.bias", "layers.0.cross_attn.value_proj.weight"),
    "SalienceTransformer._ratios_host": (
        lambda: pkg.SalienceTransformer(_encoder(), num_classes=11, layer_filter_ratio=(1.0, 0.6)),
        lambda m: m._ratios_host(), "layer_filter_ratio", "level_filter_ratio"),
    "MultiScaleDeformableAttention.fused_projection": (lambda: pkg.MultiScaleDeformableAttention(256, 4, 8, 4),
                                                       lambda m: m.fused_projection(), "attention_weights.bias",
                                                       "sampling_offsets.weight"),
}


@pytest.mark.parametrize("change", CHANGES)
@pytest.mark.parametrize("site", list(CPU_SITES))
def test_site_rebuilds_after_a_source_changes(site, change):
    make, read, replaced, viewed = CPU_SITES[site]
    _check_site(make(), read, replaced, viewed, change)


# ---- the sites that build with kernels ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("change", CHANGES)
@pytest.mark.parametrize("split", ["split_weight", "split_weight_pair", "split_weight_f16", "_train_splits"])
def test_gemm_weight_split_rebuilds_after_the_weight_changes(split, change):
    fn = getattr(pkg.gemm, split)
    _check_site(nn.Linear(256, 256).to(DEV), lambda m: fn(m.weight), "weight", "weight", change)


@pytest.mark.gpu
@pytest.mark.parametrize("change", CHANGES)
def test_neck_kernel_weights_rebuild_after_a_source_changes(change):
    net = pkg.RepVGGPluXNetwork([256] * 4, [256] * 4, groups=4, norm_layer=nn.BatchNorm2d, activation=nn.SiLU).to(DEV).eval()
    _check_site(net, lambda m: m._kernel_weights(), "lateral_convs.0.1.running_var", "lateral_convs.0.0.weight", change)


@pytest.mark.gpu
@pytest.mark.parametrize("change", CHANGES)
def test_channel_mapper_kernel_weights_rebuild_after_a_source_changes(change):
    mapper = pkg.ChannelMapper([256, 256], 256, 3).to(DEV).eval()
    _check_site(mapper, lambda m: m._kernel_weights(), "convs.1.1.bias", "convs.0.0.weight", change)
