"""Training-step benchmark under torch.use_deterministic_algorithms(True): bench.py's `--mode train` measurement, unchanged,
with torch's deterministic mode on -- the bit-reproducible MSDA and score-upsample backwards, still captured in one CUDA graph.

    python tools/bench_train_deterministic.py [--steps K --warmup W ...]   # any bench.py option; --mode train is implied

Sets CUBLAS_WORKSPACE_CONFIG=:4096:8 when it is unset (torch raises without it in deterministic mode; it must be set before the
first cuBLAS call) and prints bench.py's JSON result line with "deterministic": true added to its "config"."""
import json
import os
import sys

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import torch  # noqa: E402

torch.use_deterministic_algorithms(True)

import bench  # noqa: E402

_emit = bench.emit


def _emit_marked(line: str):
    result = json.loads(line)
    result.setdefault("config", {})["deterministic"] = True
    _emit(json.dumps(result))


bench.emit = _emit_marked
sys.argv = [os.path.join(ROOT, "bench.py"), "--mode", "train", *sys.argv[1:]]
bench.main()
