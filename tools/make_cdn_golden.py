"""Writes tests/golden/cdn_queries.npz from the UNMODIFIED reference GenerateCDNQueries (models/bricks/denoising.py) on the CPU.
Needs SDETR_REFERENCE_ROOT.

The reference's util/misc.py imports accelerate; the stub module for it holds the reference's own ``inverse_sigmoid``, taken
from that file's source.  Per case (oracle.denoising.CASES, inputs regenerated from the stored seed): the module's weights
after ``torch.manual_seed(seed)``, the random tensors its forward draws (recorded in call order by wrapping
``torch.rand_like`` / ``torch.randint_like`` around the call), the five outputs, and ``label_encoder.weight.grad`` for the
upstream gradient ``randn(label_queries.shape)`` of a generator seeded with seed + 1.  Also the state_dict of a module
constructed under ``torch.manual_seed(oracle.denoising.INIT["seed"])``.

    SDETR_REFERENCE_ROOT=/path/to/Salience-DETR python tools/make_cdn_golden.py
"""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import denoising as odn  # noqa: E402

SEED = 40


def load_reference():
    ref = os.environ.get("SDETR_REFERENCE_ROOT", "")
    if not os.path.isfile(os.path.join(ref, "models", "bricks", "denoising.py")):
        raise SystemExit("set SDETR_REFERENCE_ROOT to a checkout of the reference")
    sys.path.insert(0, ref)
    src = open(os.path.join(ref, "util", "misc.py")).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "inverse_sigmoid")
    misc = types.ModuleType("util.misc")
    misc.torch = torch
    exec(compile(ast.Module(body=[fn], type_ignores=[]), "util/misc.py", "exec"), misc.__dict__)
    pkg = types.ModuleType("util")
    pkg.__path__ = [os.path.join(ref, "util")]
    pkg.misc = misc
    sys.modules["util"], sys.modules["util.misc"] = pkg, misc
    from models.bricks.denoising import GenerateCDNQueries
    return GenerateCDNQueries


class record_draws:
    """Records every tensor torch.rand_like / torch.randint_like return while active, in call order."""

    def __enter__(self):
        self.draws, self.saved = [], (torch.rand_like, torch.randint_like)

        def wrap(f):
            def g(*a, **k):
                t = f(*a, **k)
                self.draws.append(t.clone())
                return t
            return g
        torch.rand_like, torch.randint_like = wrap(self.saved[0]), wrap(self.saved[1])
        return self

    def __exit__(self, *exc):
        torch.rand_like, torch.randint_like = self.saved


def main():
    Ref = load_reference()
    arrays = {"seed": np.array(SEED)}
    torch.manual_seed(odn.INIT["seed"])
    m = Ref(*odn.INIT["cfg"])
    for k, v in m.state_dict().items():
        arrays["init." + k] = v.numpy()
    for ci, name in enumerate(odn.CASES):
        seed = SEED + ci
        labels, boxes, cfg = odn.case_inputs(name, seed)
        torch.manual_seed(seed)
        m = Ref(*cfg)
        arrays[f"{name}.weight"] = m.label_encoder.weight.detach().numpy().copy()
        with record_draws() as rec:
            lq, bq, mask, groups, max_gt = m(labels, boxes)
        names = (["label_rand", "label_randint"] if cfg[4] * 0.5 > 0 else []) + (["box_randint", "box_rand"] if cfg[5] > 0 else [])
        assert len(rec.draws) == len(names), (name, len(rec.draws))
        for n, t in zip(names, rec.draws):
            arrays[f"{name}.{n}"] = t.numpy()
        up = torch.randn(lq.shape, generator=torch.Generator().manual_seed(seed + 1))
        if lq.requires_grad:
            (lq * up).sum().backward()
            arrays[f"{name}.weight_grad"] = m.label_encoder.weight.grad.numpy()
        else:  # no gt at all: nothing reaches the embedding
            arrays[f"{name}.weight_grad"] = np.zeros_like(arrays[f"{name}.weight"])
        arrays[f"{name}.label_queries"] = lq.detach().numpy()
        arrays[f"{name}.box_queries"] = bq.numpy()
        arrays[f"{name}.attn_mask"] = mask.numpy()
        arrays[f"{name}.groups"], arrays[f"{name}.max_gt"] = np.array(groups), np.array(max_gt)
    path = os.path.join(ROOT, "tests", "golden", "cdn_queries.npz")
    np.savez_compressed(path, **arrays)
    print(path, "bytes", os.path.getsize(path))


if __name__ == "__main__":
    main()
