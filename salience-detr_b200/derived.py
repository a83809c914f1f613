"""Tensors derived from parameters (weight splits, transposes, concatenations, folded convolutions), cached until a source
changes.

The kernels never take an ``nn.Parameter`` as it stands; they take a tensor built from one or more of them.  ``cached`` keeps
that tensor per ``(owner, name)`` and rebuilds it when a source tensor is a different object, was modified in place (its
version counter moved), or now has another data pointer, shape or strides (``p.data = ...`` swapped in another view, even of
the same storage).  Owners and sources are held weakly: an owner that is freed drops its entries.  A cached value must not
reference its owner, or the owner is never freed.
"""
from __future__ import annotations

import weakref
from typing import Callable, Dict, Hashable, Sequence, TypeVar

import torch
from torch import Tensor

T = TypeVar("T")

# id(owner) -> (weak reference to the owner, {name: (weak references to the sources, their stamps, value)}).  The reference's
# callback drops the entry as the owner is freed, before its id can be reused.  A plain dict keyed by id() because every
# projection of an eager forward looks its weights up here: WeakIdKeyDictionary builds a key object per lookup, which costs
# about twice as much.
_entries: Dict[int, tuple] = {}


def cached(owner, name: Hashable, sources: Sequence[Tensor], build: Callable[[], T]) -> T:
    """The value ``build()`` (run under ``torch.no_grad()``) made for ``(owner, name)`` from ``sources``: the same object while
    no source has changed, else a new one, which replaces it."""
    slot = _entries.get(id(owner))
    if slot is None or slot[0]() is not owner:
        key = id(owner)
        slot = _entries[key] = (weakref.ref(owner, lambda _, key=key, pop=_entries.pop: pop(key, None)), {})
    stamps = [(s._version, s.data_ptr(), s.shape, s.stride()) for s in sources]
    hit = slot[1].get(name)
    if hit is not None and hit[1] == stamps and all(r() is s for r, s in zip(hit[0], sources)):
        return hit[2]
    with torch.no_grad():
        value = build()
    slot[1][name] = ([weakref.ref(s) for s in sources], stamps, value)
    return value
