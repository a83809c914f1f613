import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """-> (arrays dict of torch tensors, state_dict) from tests/golden/<name>.npz"""
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    arrs, sd = {}, {}
    for k in z.files:
        if z[k].dtype.kind in "US":
            continue
        t = torch.from_numpy(z[k])
        if k.startswith("sd."):
            sd[k[3:]] = t
        else:
            arrs[k] = t
    return arrs, sd


TINY_CFG = dict(heads=2, points=4, topk_sa=20, num_layers=3, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
                layer_filter_ratio=(1.0, 0.6, 0.3))


@pytest.fixture(scope="session", autouse=True)
def _poison_device_memory():
    """SDETR_POISON=<hex byte>: fill the caching allocator's memory with a byte pattern before the GPU tests, so a
    kernel that reads memory the path never wrote sees NaNs / wild indices instead of stale-but-plausible data."""
    pat = os.environ.get("SDETR_POISON")
    if pat and torch.cuda.is_available():
        free, _ = torch.cuda.mem_get_info()
        big = [torch.empty(int(free * 0.3), dtype=torch.uint8, device="cuda:0").fill_(int(pat, 16)) for _ in range(3)]
        small = [torch.empty(s, dtype=torch.uint8, device="cuda:0").fill_(int(pat, 16))
                 for s in (512, 4096, 65536, 524288, 1 << 20) for _ in range(400)]
        torch.cuda.synchronize()
        del big, small
    if os.environ.get("SDETR_TRACE_NAN"):
        from tools import nan_trace
        nan_trace.install()
    yield


C256_CFG = dict(heads=8, points=4, topk_sa=64, num_layers=2, level_filter_ratio=(0.4, 0.8, 1.0, 1.0),
                layer_filter_ratio=(1.0, 0.5))


def load_c256_golden():
    """tests/golden/encoder_c256.npz (made by oracle/make_golden.py from the reference at its real width): returns
    (arrays, state_dict, (feats, masks, pos)) with the weights / inputs regenerated from their seeds."""
    import json
    from oracle import oracle as orc
    z = np.load(os.path.join(GOLDEN, "encoder_c256.npz"), allow_pickle=False)
    shapes = json.loads(str(z["shapes_json"]))
    arrs = {k: torch.from_numpy(z[k]) for k in z.files if k != "shapes_json"}
    sd = orc.deterministic_state_dict(shapes, 11)
    inputs = orc.synthetic_inputs([(384, 512), (384, 512)], (384, 512), 256, seed=11)
    return arrs, sd, inputs
