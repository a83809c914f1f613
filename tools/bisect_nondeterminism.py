"""Debug aid: hash the outputs of every C-ABI wrapper / GEMM call inside the encoder half and report the first call
whose output differs between repeated runs on identical inputs."""
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import salience_detr_b200 as pkg
from salience_detr_b200 import cabi, gemm
from salience_detr_b200.synthetic import build_model, make_inputs

dev = torch.device("cuda:0")
config = sys.argv[1] if len(sys.argv) > 1 else "resnet50_5scale_bs2"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
LOG = []


def digest(x):
    outs = x if isinstance(x, (tuple, list)) else (x,)
    d = []
    for t in outs:
        if torch.is_tensor(t) and t.is_cuda and t.numel():
            c = t.contiguous()
            if c.dtype in (torch.float32, torch.int32):
                v = c.view(torch.int32).to(torch.int64)
            elif c.dtype == torch.int64:
                v = c
            else:
                v = c.to(torch.int64)
            v = v.flatten()
            d.append((int(v.sum().item()), int((v * (torch.arange(v.numel(), device=dev) % 1021 + 1)).sum().item())))
    return tuple(d)


def wrap(mod, name):
    fn = getattr(mod, name)

    def inner(*a, **kw):
        out = fn(*a, **kw)
        shapes = [tuple(t.shape) for t in a if torch.is_tensor(t)]
        LOG.append((name, shapes, digest(out if out is not None else a[0])))
        return out
    setattr(mod, name, inner)


for name in ("token_gather", "class_max_times_fg", "topk_desc", "rows_gather_add", "add_layernorm", "rows_scatter_",
             "token_scatter_", "background_embed_", "msda_fused_forward", "salience_select", "order_prefixes",
             "flatten_tokens", "zero_masked_rows_", "score_modulate_"):
    if hasattr(cabi, name):
        wrap(cabi, name)
wrap(gemm, "linear")
wrap(F, "linear")
wrap(F, "scaled_dot_product_attention")

strides = (4, 8, 16, 32) if "5scale" in config else (8, 16, 32)
model = build_model(strides=strides).to(dev)
feats, masks, pos = make_inputs(config, seed=1, device=dev)
first = None
for r in range(reps):
    LOG.clear()
    with torch.no_grad():
        model.forward_encoder(feats, masks, pos)
    cur = list(LOG)
    if first is None:
        first = cur
        print("calls per forward:", len(cur), flush=True)
        continue
    for i, (a, b) in enumerate(zip(first, cur)):
        if a != b:
            print("rep", r, "first differing call #%d:" % i, b[0], b[1], flush=True)
            print("   previous call:", first[i - 1][0], first[i - 1][1], flush=True)
            break
    else:
        print("rep", r, "identical", flush=True)
